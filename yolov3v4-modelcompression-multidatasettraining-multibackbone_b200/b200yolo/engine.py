"""Graph executor for Darknet models on sm_90a.

Replaces the reference's per-module Python loop (models.py:508-561, ~250-520 ATen/cuDNN launches per forward)
by a static plan over NHWC fp16 buffers:

  * conv + folded BN + activation (+ the following Shortcut) = one wgmma implicit-GEMM launch,
  * route/concat is zero-copy: producers write straight into their channel slot of the concat buffer,
  * the stem reads the NCHW fp32 image directly, the head convs emit fp32 for the decode kernel,
  * the launch sequence is captured once into a CUDA graph per input shape and replayed.

Parameters stay in the nn.Module tree (fp32, NCHW) and are folded/packed on the device whenever they change.
"""
import os

import torch
import torch.nn as nn

from . import ops
from .lib import WLAYOUT_S2_PAIRS

_ACT_OF_CLASS = {'LeakyReLU': 'leaky', 'Mish': 'mish', 'ReLU6': 'relu6', 'HardSwish': 'h_swish', 'ReLU': 'relu',
                 'Swish': 'swish'}


class LazyFeatures(list):
    """feature_out of the reference API (models.py:542-543): one entry per conv block that does not feed a YOLO layer.
    Entries are materialised (NHWC fp16 -> NCHW fp32) on access; they alias engine buffers and are only valid
    until the next forward."""

    def __init__(self, views):
        super().__init__([None] * len(views))
        self._views = views

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        v = self._views[i]
        if v is None:
            raise RuntimeError("feature_out[%d] was not kept: set model.keep_features = True before the forward" % i)
        return ops.nhwc_to_nchw(v)

    def __iter__(self):
        return (self[i] for i in range(len(self)))


class _Tensor:
    """Logical activation tensor: NHWC view = buffer[..., c0:c0+C]."""
    __slots__ = ('C', 'H', 'W', 'buf', 'c0', 'dtype')

    def __init__(self, C, H, W, dtype=torch.float16):
        self.C, self.H, self.W, self.dtype = C, H, W, dtype
        self.buf, self.c0 = None, 0

    def view(self):
        return self.buf[..., self.c0:self.c0 + self.C]

    def view_k(self):
        """View for a tensor-core consumer: the channel count rounded up to 16 (the MMA K granule is 16 fp16 elements).
        MobileNet widths (24, 40, 72, 120, 184, 200) are not: their buffers are allocated zero-filled with a pitch that
        is a multiple of 16 and nobody ever writes the pad channels, the packed weights carry zero columns there (a
        tensor living inside a concat buffer may see its neighbour's channels instead of zeros: finite values times
        zero weights)."""
        ck = (self.C + 15) // 16 * 16
        if ck == self.C:
            return self.view()
        if self.c0 + ck > self.buf.shape[3]:
            raise RuntimeError("activation buffer too narrow for the padded channel view (C=%d)" % self.C)
        return self.buf[..., self.c0:self.c0 + ck]


def _block_parts(block):
    """nn.Sequential conv block -> (conv, bn or None, activation name, slope)."""
    conv, bn, act, slope = None, None, 'linear', 0.1
    for m in block:
        name = m.__class__.__name__
        if isinstance(m, nn.Conv2d):
            conv = m
        elif isinstance(m, nn.BatchNorm2d):
            bn = m
        elif name in _ACT_OF_CLASS:
            act = _ACT_OF_CLASS[name]
            if name == 'LeakyReLU':
                slope = m.negative_slope
    return conv, bn, act, slope


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
    version.  Entries are keyed (layer index, layout): the pixel-pair layouts depend on the plan (an odd width rules
    them out), the base layout does not."""

    def __init__(self):
        self.version = None
        self.packs = {}


class Plan:
    def __init__(self, model, x_shape, device, training, keep_features=False, store=None, shared_weights=None):
        if training:
            raise NotImplementedError("training plan is built by b200yolo.train_engine")
        self.model = model
        self.keep_features = bool(keep_features)
        self.device = device
        self.B, self.Cin, self.H, self.W = x_shape
        self.store = store if store is not None else SlotStore(device)
        self.shared_weights = shared_weights if shared_weights is not None else EvalWeights()
        self.held = {}          # slot name -> version taken
        self.steps = []
        self.wkey = {}          # layer index -> key of its packed weights in shared_weights.packs
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
        pitch = (C + 15) // 16 * 16
        return self._take(('act', name, pitch, torch.float16), (self.B, H, W, pitch))

    def _w(self, i):
        return self.shared_weights.packs[self.wkey[i]]

    def _stem_workspace(self, conv):
        d = ops.make_conv_desc((self.B, self.H, self.W, conv.in_channels), conv.in_channels, conv.out_channels,
                               conv.kernel_size[0], conv.stride[0], conv.padding[0], conv.out_channels)
        return self._take(('stem_ws',), (ops.stem_workspace_bytes(d) // 2,))

    # ---------------------------------------------------------------------------------------------------------
    def _build(self):
        model, B = self.model, self.B
        defs, mods, routs = model.module_defs, model.module_list, model.routs
        n = len(defs)
        dev = self.device

        # 1) shapes
        shapes = []  # (C,H,W) of every layer output
        prev = (self.Cin, self.H, self.W)
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            C, H, W = prev
            if t in ('convolutional', 'depthwise'):
                conv = _block_parts(m)[0]
                k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
                H, W = ops.conv_out_hw(H, W, k, s, p)
                C = conv.out_channels
            elif t == 'se':
                pass
            elif t == 'maxpool':
                k, s = d['size'], d['stride']
                if k == 2 and s == 1:
                    H, W = (H + 1 - k) // s + 1, (W + 1 - k) // s + 1
                else:
                    p = (k - 1) // 2
                    H, W = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
            elif t == 'upsample':
                H, W = H * d['stride'], W * d['stride']
            elif t == 'route':
                srcs = [i + l if l < 0 else l for l in d['layers']]
                C = sum(shapes[s][0] for s in srcs)
                if 'groups' in d:
                    C //= 2
                H, W = shapes[srcs[0]][1], shapes[srcs[0]][2]
            elif t in ('shortcut', 'yolo'):
                pass
            else:
                raise NotImplementedError("layer type '%s' is not supported by the sm_90a engine yet" % t)
            prev = (C, H, W)
            shapes.append(prev)

        # 2) fusion decisions
        is_head = [False] * n       # conv directly followed by a yolo layer -> fp32 output
        fused_into = [None] * n     # shortcut i fused into conv i-1
        for i, d in enumerate(defs):
            if d['type'] == 'yolo' and i > 0 and defs[i - 1]['type'] == 'convolutional':
                is_head[i - 1] = True
            if d['type'] == 'shortcut' and i > 0:
                frm = [i + l if l < 0 else l for l in d['from']]
                if (not self.keep_features  # feature_out must expose the conv output *before* the add
                        and len(frm) == 1 and defs[i - 1]['type'] == 'convolutional' and not routs[i - 1]
                        and not getattr(mods[i], 'weight', False) and shapes[frm[0]] == shapes[i - 1]
                        and shapes[i - 1][0] % 8 == 0 and i - 1 > 0):
                    fused_into[i] = i - 1

        # 3) logical tensors; aliases for single-source routes
        tens = [None] * n
        for i, d in enumerate(defs):
            t = d['type']
            if t == 'yolo':
                continue
            if t == 'route' and len(d['layers']) == 1 and 'groups' not in d:
                continue  # alias, resolved below
            C, H, W = shapes[i]
            tens[i] = _Tensor(C, H, W, torch.float32 if is_head[i] else torch.float16)
        for i, d in enumerate(defs):
            if fused_into[i] is not None:
                tens[fused_into[i]] = tens[i]  # the conv writes the shortcut's output tensor
        alias = {}
        for i, d in enumerate(defs):
            if d['type'] == 'route' and len(d['layers']) == 1 and 'groups' not in d:
                l = d['layers'][0]
                src = i + l if l < 0 else l
                while src in alias:
                    src = alias[src]
                alias[i] = src
                tens[i] = tens[src]

        # 4) concat placement: multi-source routes become pre-allocated buffers their producers write into
        placed = set()
        copies = {}  # route index -> list of (src tensor, channel offset) that must be copied
        for i, d in enumerate(defs):
            if d['type'] != 'route' or len(d['layers']) == 1:
                continue
            srcs = [i + l if l < 0 else l for l in d['layers']]
            dst = tens[i]
            dst.buf = self._new_act(('cat', i), dst.C, dst.H, dst.W)
            off = 0
            for s in srcs:
                st = tens[s]
                if (id(st) not in placed and st.buf is None and off % 8 == 0 and st.dtype == torch.float16
                        and st is not dst):
                    st.buf, st.c0 = dst.buf, off
                    placed.add(id(st))
                else:
                    copies.setdefault(i, []).append((st, off))
                off += st.C
        for i, d in enumerate(defs):  # grouped routes: upper half of the channels of the previous layer
            if d['type'] == 'route' and 'groups' in d:
                pass  # resolved at allocation time below (needs the source buffer)

        # 5) allocate what is left and emit the launch list
        def alloc(t, i):
            if t.buf is None:
                if t.dtype == torch.float16:
                    t.buf = self._new_act(i, t.C, t.H, t.W)
                else:
                    pitch = ((t.C + 3) // 4) * 4
                    t.buf = self._take(('head', i, pitch, t.dtype), (B, t.H, t.W, pitch), t.dtype)
                t.c0 = 0
            return t

        self.yolo = []
        self.feature_views = []
        row_off = 0
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            if t == 'depthwise':
                conv, bn, act, slope = _block_parts(m)
                if conv.groups != conv.in_channels or conv.out_channels != conv.in_channels:
                    raise NotImplementedError("only channel-multiplier-1 depthwise convolutions are supported")
                self.steps.append(('dw', i, tens[i - 1], alloc(tens[i], i), conv, bn, act, slope))
            elif t == 'se':
                fc = m[0].fc if isinstance(m, nn.Sequential) else m.fc
                src = tens[i - 1]
                ws = self._take(('se_ws', i), (B, 3 * src.C + fc[0].out_features), torch.float32)
                self.steps.append(('se', i, src, alloc(tens[i], i), fc[0], fc[2], ws))
            elif t == 'convolutional':
                conv, bn, act, slope = _block_parts(m)
                if conv.groups != 1:
                    raise NotImplementedError("grouped convolution is not supported by the sm_90a engine yet")
                out = alloc(tens[i], i)
                res = None
                if i + 1 < n and fused_into[i + 1] == i:
                    l = defs[i + 1]['from'][0]
                    res = tens[i + 1 + l if l < 0 else l]
                src = None if i == 0 else tens[i - 1]
                self.steps.append(('conv', i, src, out, res, conv, bn, act, slope))
            elif t == 'shortcut':
                if fused_into[i] is not None:
                    continue
                frm = [i + l if l < 0 else l for l in d['from']]
                if getattr(m, 'weight', False):
                    raise NotImplementedError("weighted shortcut is not supported by the sm_90a engine yet")
                out = alloc(tens[i], i)
                cur = tens[i - 1]
                for s in frm:
                    # widths may differ (layers.py:57-72): the sum covers the first min(nx, na) channels, the rest of x
                    # passes through
                    self.steps.append(('add', cur, tens[s], out))
                    cur = out
            elif t == 'route':
                if len(d['layers']) == 1:
                    if 'groups' in d:
                        src = tens[i - 1]
                        g = tens[i]
                        g.buf, g.c0 = src.buf, src.c0 + src.C // 2
                    continue
                for st, off in copies.get(i, []):
                    self.steps.append(('copy', st, tens[i], off))
            elif t == 'upsample':
                self.steps.append(('upsample', tens[i - 1], alloc(tens[i], i), d['stride']))
            elif t == 'maxpool':
                k, s = d['size'], d['stride']
                self.steps.append(('maxpool', tens[i - 1], alloc(tens[i], i), k, s, k == 2 and s == 1))
            elif t == 'yolo':
                raw = tens[i - 1]
                rows = m.na * raw.H * raw.W
                self.yolo.append((m, raw, row_off, rows))
                row_off += rows
        self.total_rows = row_off
        # feature_out (models.py:542-543): every nn.Sequential block whose successor is not a YOLO layer
        for i, m in enumerate(mods):
            if m.__class__.__name__ == 'Sequential' and i + 1 < n and defs[i + 1]['type'] != 'yolo':
                self.feature_views.append(tens[i] if (self.keep_features and tens[i] is not None) else None)
        self.anchors_px = [m.anchors.to(dev).float().contiguous() for (m, _, _, _) in self.yolo]

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
            if st[0] == 'dw':
                _, i, src, out, conv, bn, act, slope = st
                key = self.wkey[i] = (i, 'dw')
                if key in packs:
                    continue
                w = conv.weight.detach().float().contiguous()
                if bn is not None:           # fold: y = conv * gamma/sqrt(var+eps) + (beta - mean*gamma/sqrt(var+eps))
                    sc = (bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)).float()
                    bi = (bn.bias.detach() - bn.running_mean * sc).float()
                    if conv.bias is not None:
                        bi = bi + conv.bias.detach().float() * sc
                else:
                    sc = None
                    bi = conv.bias.detach().float().contiguous() if conv.bias is not None else None
                packs[key] = (w, sc.contiguous() if sc is not None else None,
                              bi.contiguous() if bi is not None else None)
                continue
            if st[0] != 'conv':
                continue
            _, i, src, out, res, conv, bn, act, slope = st
            layout = 'pair' if self._pair_packable(st) else 's2' if self._s2_pair_packable(st) else 'base'
            key = self.wkey[i] = (i, layout)
            if key in packs:
                continue
            bnp = None
            eps = 1e-5
            if bn is not None:
                bnp = (bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var)
                eps = bn.eps
            base = packs.get((i, 'base'))
            if base is None:
                stem = conv.in_channels <= 4
                wsrc = conv.weight.detach()
                if not stem and conv.in_channels % 16 != 0:      # zero columns for the padded K channels (view_k)
                    wsrc = torch.nn.functional.pad(wsrc, (0, 0, 0, 0, 0, (-conv.in_channels) % 16))
                wp, bias, w32 = ops.pack_conv_weights(wsrc, conv.bias.detach() if conv.bias is not None
                                                      else None, bnp, eps, want_fp32=stem)
                wstem = None
                if stem and (conv.in_channels * conv.kernel_size[0] <= 16 or
                             conv.in_channels * conv.kernel_size[0] ** 2 <= 32):
                    wstem = ops.pack_stem_weights(w32)
                base = packs[(i, 'base')] = (wp, bias, w32, wstem)
            if layout == 'pair':
                packs[key] = base + (self._pair_pack(conv, bnp, eps),)
            elif layout == 's2':
                _, bias_f, w32f = ops.pack_conv_weights(conv.weight.detach(), conv.bias.detach() if conv.bias is not None
                                                        else None, bnp, eps, want_fp32=True)
                packs[key] = base + (('s2', ops.s2_pair_weights(w32f).half(), bias_f),)

    # ---- pixel-pair packing of the Cin = 32 3x3 layers --------------------------------------------------------------
    # With 32 input channels a tap of the im2col gather is a 64-byte row: one TMA request per pixel per tap, and the
    # layer is bound by the TMA request rate (0.16 of the tensor peak, 31-46 % of HBM in round 1), not by HBM.  The NHWC
    # tensor [B,H,W,32] is the same memory as [B,H,W/2,64]: viewed as pixel PAIRS the same convolution is a 3x3 conv
    # with 64 input and 2*Cout output channels whose weights are the original taps placed at
    # s = 2(kwp-1) + i_sub - o_sub + 1 (zero elsewhere).  Half of the MACs multiply zeros, but the rows are 128 bytes,
    # the tile count halves and N = 128 brings the CTA-pair path in -- no new kernel, only a weight layout.
    def _pair_packable(self, st):
        if os.environ.get('B2Y_PAIRPACK', '1') == '0':
            return False
        _, i, src, out, res, conv, bn, act, slope = st
        if src is None or conv.kernel_size[0] != 3 or conv.stride[0] != 1 or conv.padding[0] != 1:
            return False
        if conv.in_channels != 32 or conv.out_channels > 128 or conv.out_channels % 8 or src.W % 2:
            return False
        full = lambda t: t.c0 == 0 and t.buf.shape[3] == t.C and t.dtype == torch.float16
        return full(src) and full(out) and (res is None or full(res))

    def _s2_pair_packable(self, st):
        """3x3 / stride-2 layers with 32 input channels (the first downsampling conv): B2Y_WLAYOUT_S2_PAIRS -- the input
        read as pixel pairs makes it a 3 x 2 window with stride 2 x 1 over 128-byte rows (6 im2col boxes, not 9 halves)."""
        if os.environ.get('B2Y_PAIRPACK', '1') == '0':
            return False
        _, i, src, out, res, conv, bn, act, slope = st
        if src is None or conv.kernel_size[0] != 3 or conv.stride[0] != 2 or conv.padding[0] != 1:
            return False
        if conv.in_channels != 32 or src.W % 2:
            return False
        return src.c0 == 0 and src.buf.shape[3] == src.C and src.dtype == torch.float16

    def _pair_pack(self, conv, bnp, eps):
        O, I = conv.out_channels, conv.in_channels
        _, bias, w32 = ops.pack_conv_weights(conv.weight.detach(), conv.bias.detach() if conv.bias is not None else None,
                                             bnp, eps, want_fp32=True)
        w2 = torch.zeros((2 * O, 2 * I, 3, 3), dtype=torch.float32, device=w32.device)
        for o_sub in range(2):
            for i_sub in range(2):
                for kwp in range(3):
                    s_ = 2 * (kwp - 1) + i_sub - o_sub + 1
                    if 0 <= s_ <= 2:
                        w2[o_sub * O:(o_sub + 1) * O, i_sub * I:(i_sub + 1) * I, :, kwp] = w32[:, :, :, s_]
        wp2, _, _ = ops.pack_conv_weights(w2)
        return wp2, torch.cat([bias, bias]).contiguous()

    def _launch_all(self, x):
        for st in self.steps:
            kind = st[0]
            if kind == 'conv':
                _, i, src, out, res, conv, bn, act, slope = st
                wp, bias, w32, wstem = self._w(i)[:4]
                k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
                if src is None:
                    if conv.in_channels > 4:
                        raise NotImplementedError("first layer with more than 4 input channels")
                    if wstem is not None and wstem.dim() == 2 and conv.out_channels <= 64:
                        # full-im2col weight layout: the fused kernel builds the A tile in smem (no workspace)
                        ops.stem_conv_fused(x, wstem, bias, k, s, p, act=act, slope=slope, out=out.view(),
                                            x_div=256.0 if x.dtype == torch.uint8 else 1.0)
                    elif wstem is not None:
                        if x.dtype != torch.float32:
                            x = x.float() / 256.0 if x.dtype == torch.uint8 else x.float()
                        if getattr(self, 'stem_ws', None) is None:
                            self.stem_ws = self._stem_workspace(conv)
                        ops.stem_conv_tc(x, wstem, bias, conv.in_channels, k, s, p, act=act, slope=slope,
                                         out=out.view(), workspace=self.stem_ws)
                    else:
                        if x.dtype != torch.float32:
                            x = x.float() / 256.0 if x.dtype == torch.uint8 else x.float()
                        ops.stem_conv(x, w32, bias, k, s, p, act=act, slope=slope, out=out.view())
                elif len(self._w(i)) == 5 and isinstance(self._w(i)[4][0], str):
                    _, wps2, bias_s2 = self._w(i)[4]
                    ops.conv2d(src.view(), wps2, bias_s2, k, s, p, act=act, slope=slope,
                               residual=res.view() if res is not None else None, out=out.view(),
                               w_layout=WLAYOUT_S2_PAIRS)
                elif len(self._w(i)) == 5:
                    wp2, bias2 = self._w(i)[4]
                    pairs = lambda t: t.buf.view(t.buf.shape[0], t.H, t.W // 2, 2 * t.C)
                    ops.conv2d(pairs(src), wp2, bias2, 3, 1, 1, act=act, slope=slope,
                               residual=pairs(res) if res is not None else None, out=pairs(out))
                else:
                    ops.conv2d(src.view_k(), wp, bias, k, s, p, act=act, slope=slope,
                               residual=res.view() if res is not None else None, out=out.view())
            elif kind == 'dw':
                _, i, src, out, conv, bn, act, slope = st
                w, sc, bi = self._w(i)
                ops.dwconv2d(src.view(), w, conv.kernel_size[0], conv.stride[0], conv.padding[0], scale=sc, bias=bi,
                             act=act, slope=slope, out=out.view())
            elif kind == 'se':
                _, i, src, out, fc1, fc2, ws = st
                ops.se_fwd(src.view(), fc1.weight.detach(), fc2.weight.detach(), out=out.view(), ws=ws)
            elif kind == 'add':
                xv, av, ov = st[1].view(), st[2].view(), st[3].view()
                n = min(xv.shape[3], av.shape[3])
                ops.add(xv[..., :n], av[..., :n], out=ov[..., :n])
                if xv.shape[3] > n and st[1] is not st[3]:
                    ops.copy_channels(xv[..., n:], ov[..., n:])
            elif kind == 'copy':
                _, srct, dst, off = st
                ops.copy_channels(srct.view(), dst.buf[..., off:off + srct.C])
            elif kind == 'upsample':
                ops.upsample(st[1].view(), st[3], out=st[2].view())
            elif kind == 'maxpool':
                ops.maxpool(st[1].view(), st[3], st[4], tiny_pad=st[5], out=st[2].view())
        for (m, raw, row_off, rows), anc in zip(self.yolo, self.anchors_px):
            ops_io = self.io
            _, p = ops.yolo_decode(raw.buf, m.na, m.no, anc, m.stride, io=ops_io, row_offset=row_off)
            self.p_out.append(p)

    # ---- measurement helpers (bench.py) -----------------------------------------------------------------------
    def _launch_step(self, st, x):
        saved = self.steps
        self.steps = [st]
        yolo = self.yolo
        self.yolo = []
        try:
            self._launch_all(x)
        finally:
            self.steps, self.yolo = saved, yolo

    def launches_per_forward(self):
        return len(self.steps) + len(self.yolo) + (1 if getattr(self, 'stem_ws', None) is not None else 0)

    def step_info(self, st):
        """(label, algorithmic FLOPs, algorithmic HBM bytes) of one launch."""
        kind = st[0]
        B = self.B
        if kind == 'conv':
            _, i, src, out, res, conv, bn, act, slope = st
            k = conv.kernel_size[0]
            M = B * out.H * out.W
            flops = 2.0 * M * conv.out_channels * conv.in_channels * k * k
            in_hw = (self.H * self.W) if src is None else (src.H * src.W)
            in_bytes = B * in_hw * conv.in_channels * (4 if src is None else 2)
            out_bytes = M * conv.out_channels * (4 if out.dtype == torch.float32 else 2)
            w_bytes = conv.out_channels * conv.in_channels * k * k * 2
            res_bytes = M * conv.out_channels * 2 if res is not None else 0
            label = "L%03d conv %dx%d s%d %d->%d @%dx%d %s%s" % (i, k, k, conv.stride[0], conv.in_channels,
                                                                 conv.out_channels, out.H, out.W, act,
                                                                 "+res" if res is not None else "")
            return label, flops, in_bytes + out_bytes + w_bytes + res_bytes, src is None
        t_in, t_out = st[1], (st[3] if kind == 'add' else st[2])
        if kind == 'copy':
            n = B * st[1].H * st[1].W * st[1].C * 2
            return "copy C=%d @%dx%d" % (st[1].C, st[1].H, st[1].W), 0.0, 2 * n, False
        n_in = B * t_in.H * t_in.W * t_in.C * 2
        n_out = B * t_out.H * t_out.W * t_out.C * 2
        if kind == 'add':
            n_in *= 2
        return "%s C=%d @%dx%d" % (kind, t_out.C, t_out.H, t_out.W), 0.0, n_in + n_out, False

    def profile_layers(self, x, reps=10):
        """Per-launch CUDA-event timing.  Each step is captured `reps` times back to back in its own CUDA graph and the
        replay is timed (best of 3), so the CPU launch cost of eager calls (tensor-map encodes, ctypes) is excluded;
        consecutive launches of one layer re-use its tensors, so layers whose working set fits the 50 MB L2 are
        measured L2-warm (like in the real graph, where the producer layer just wrote them)."""
        x = x.contiguous()
        if self.param_version is None:
            self.forward(x)
        rows = []
        self.io = torch.empty((self.B, self.total_rows, self.yolo[0][0].no), dtype=torch.float32, device=self.device)
        for st in self.steps:
            label, flops, nbytes, is_stem = self.step_info(st)
            self._launch_step(st, x)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(reps):
                    self._launch_step(st, x)
            g.replay()
            best = None
            for _ in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                e1.synchronize()
                ms = e0.elapsed_time(e1) / reps
                best = ms if best is None else min(best, ms)
            ms = best
            rows.append({"label": label, "ms": ms, "tflops": flops / ms / 1e9 if ms > 0 else 0.0,
                         "gbs": nbytes / ms / 1e6 if ms > 0 else 0.0, "flops": flops, "bytes": nbytes,
                         "kind": "stem" if is_stem else st[0]})
            del g
        return rows

    def time_tc_convs(self, x, iters=5):
        """Time only the wgmma conv launches of one forward, back to back on the current stream.
        Returns (ms per forward-worth of conv launches, algorithmic FLOPs of those launches, n launches)."""
        x = x.contiguous().float()
        if self.param_version is None:
            self.forward(x)
        convs = [st for st in self.steps if st[0] == 'conv' and st[2] is not None]
        flops = sum(self.step_info(st)[1] for st in convs)
        saved, yolo = self.steps, self.yolo
        self.steps, self.yolo = convs, []
        try:
            self._launch_all(x)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                self._launch_all(x)
            e1.record()
            e1.synchronize()
        finally:
            self.steps, self.yolo = saved, yolo
        return e0.elapsed_time(e1) / iters, flops, len(convs)

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
        feats = LazyFeatures([None if t is None else t.view() for t in self.feature_views])
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
        key = (tuple(x.shape), bool(model.training), x.device.index, keep, x.dtype)
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
        owner = store.pinned_by()
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
                plan = TrainPlan(model, tuple(x.shape), x.device, keep, store, self.train_shared)
            else:
                plan = Plan(model, tuple(x.shape), x.device, False, keep, store, self.eval_weights)
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
