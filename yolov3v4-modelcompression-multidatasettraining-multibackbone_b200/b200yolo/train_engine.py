"""Training-mode executor: forward with batch-statistics BatchNorm and the full backward pass on sm_90a.

Replaces autograd over ~500 ATen/cuDNN calls (reference train.py:380-441 -> models.py:508-551) by a static plan:

  forward   conv (wgmma, per-channel sum / sum^2 from the epilogue) -> BatchNorm finalize + act(+shortcut) apply
  backward  yolo permute^T -> [bn+act backward reduce / apply -> wgrad (wgmma, pixel-K GEMM) -> dgrad (wgmma)]

Activations z (raw conv output) and y (post activation) are kept in NHWC fp16 (accurate forward).  Gradients w.r.t.
activations (dY) are stored in **bf16** (fp32 range: their magnitude drifts by orders of magnitude across ~100
BatchNorm layers, which fp16 cannot hold with one loss scale).  The conv data gradient dZ, which is an operand of the
two tensor-core GEMMs (dgrad with the fp16 weights, wgrad with the fp16 activations), is written in fp16 times a
per-layer power-of-two scale chosen inside the BN-backward kernel from a bound on max|dZ| (wgmma takes one 16-bit format for
both operands); the GEMM epilogues read 1/scale from device memory, so there is no host synchronisation.
Weight / BN gradients are accumulated and stored in fp32.
The plan plugs into autograd as ONE torch.autograd.Function whose inputs are the model parameters, so
loss.backward(), DistributedDataParallel hooks and torch optimisers work unchanged.
"""
import ctypes as C

import os
import weakref

import torch
import torch.nn as nn

from . import ops
from .engine import LazyFeatures, SlotStore, _pad_rows, launch_pointwise, pointwise_steps
from .layout import (STEM_WGRAD_MAX_TAPS, _Tensor, _block_parts, build_layout, feature_slots, infer_shapes, pitch,
                     sources, stem_path)
from .lib import ACT, ConvDesc, OUT_F16, call, ptr, stream_ptr

GDT = torch.bfloat16   # gradient tensors: bf16 (range of fp32) -- fp16 over/underflows across ~100 BN layers


def _round_up(v, m):
    return (v + m - 1) // m * m


def head_width(cout):
    """Output channels a YOLO head conv runs with: Cout rounded up to the K granule (16) of the data-gradient GEMM,
    at least 256.  The pad channels are zero rows of the weights and zero columns of the head gradient.  The 256 floor
    keeps every head of up to 256 filters (255 for 80 classes, 18 for one) on the layout it has always had."""
    return max(256, _round_up(cout, 16))


def _meta(shape, dtype):
    """Placeholder for a buffer that TrainPlan._carve places in an arena."""
    return torch.empty(shape, dtype=dtype, device='meta')


def _widen(view, channels):
    """The same NHWC view with `channels` channels (its buffer is at least that wide and zero beyond the view)."""
    B, H, W, C = view.shape
    return torch.as_strided(view, (B, H, W, channels), view.stride(), view.storage_offset())


class _ConvRec:
    """stem: None, or the first layer's path (layout.stem_path), which runs both its forward and its weight gradient:
    'im2col' as GEMMs over one im2col workspace, 'direct' on CUDA cores."""
    __slots__ = ('i', 'conv', 'bn', 'act', 'slope', 'src', 'z', 'y', 'res', 'head', 'stem', 'k', 's', 'p', 'Cout',
                 'Cpad', 'w16', 'wT', 'stats', 'ones', 'zeros', 'w32', 'aux_row', 'wstem', 'save', 'sums', 'dw',
                 'depthwise', 'Ipad', 'dwg', 'col_map', 'wdw', 'cidx')

    def __init__(self):
        for k in self.__slots__:
            setattr(self, k, None)


class _SeRec:
    __slots__ = ('i', 'src', 'y', 'fc1', 'fc2', 'ws', 'ws_bwd', 'w1', 'w2', 'cidx')

    def __init__(self, *fields):
        for k in self.__slots__:
            setattr(self, k, None)
        for k, v in zip(self.__slots__, fields):
            setattr(self, k, v)


class TrainShared:
    """Training state of one model that does not depend on the input shape, shared by its plans of every shape: the
    packed fp16 weights and data-gradient slabs (`w16`, `wT`) and the stem's packed weights, keyed by layer index, with
    their pack tables; the input-column maps of the layers behind a gapped concat (`col_maps`), which those tables point
    to and so must live as long as they do; the OIHW fp32 gradient outputs of the plain-autograd path; and the side
    stream of the weight gradients, so that one split-K workspace (`stream_ws`, keyed by stream) serves every plan."""

    def __init__(self, device):
        self.device = device
        self.w16, self.wT, self.wstem = {}, {}, {}
        self.col_maps = {}
        self.pack_tables = {}
        self.own_grads = {}
        self.side_stream = None


class _Pin:
    """Holds a SlotStore for one training forward until its backward has run or its autograd graph is freed.  The
    step's autograd node owns the pin; the store only keeps a weak reference, so freeing the graph frees the pin."""

    def __init__(self, store, plan):
        self.store, self.plan = store, plan
        store.pin = weakref.ref(self)

    def release(self):
        if self.store.pin is not None and self.store.pin() is self:
            self.store.pin = None


class TrainPlan:
    """The forward binds activations at their physical widths (layout.phys_width), packs weights with zero pad rows and
    input columns scattered through the source's channel map, and tells the BatchNorm apply the logical width.

    forward_only: the plan without its backward state, for a train-mode forward that records no graph (batch
    statistics and the running-statistics update).  It runs every width the eval plan runs; the gradient plan refuses
    BatchNorm widths its backward kernels cannot take.  Its slots and packed weights are its own (named ('fo', ...)), so
    a gradient-free forward between a training forward and its backward leaves everything that step saved untouched."""

    def __init__(self, model, x_shape, device, keep_features=False, store=None, shared=None, *, forward_only=False):
        self.model = model
        self.device = device
        self.keep_features = bool(keep_features)
        self.forward_only = bool(forward_only)
        self._tag = ('fo',) if self.forward_only else ()
        self.B, self.Cin, self.H, self.W = x_shape
        self.store = store if store is not None else SlotStore(device)
        self.shared = shared if shared is not None else TrainShared(device)
        self.held = {}          # slot name -> version taken
        self.convs = []
        self.order = []        # forward step list
        self.param_version = None
        self._build()

    def _take(self, name, shape, dtype):
        name = self._tag + tuple(name)
        t = self.store.take(name, shape, dtype)
        self.held[name] = self.store.versions[name]
        return t

    def _key(self, i):
        """TrainShared key of layer i's packed weights (the forward-only plans pack their own)."""
        return self._tag + (i,) if self._tag else i

    def _new_buf(self, name, Cc, H, W, dtype=torch.float16):
        # fp16: MobileNet widths (24, 40, 72 ...) get a pitch rounded up to the MMA K granule, pad channels stay zero
        # forever (slots are zero-filled and the pitch depends on the width only)
        pc = pitch(Cc, dtype)
        return self._take((name, pc, dtype), (self.B, H, W, pc), dtype)

    def _carve(self, name, fields, last=()):
        """ONE slot `name` for every meta placeholder that the (holder, attribute) pairs `fields` hold, each at a 256-byte
        aligned offset; every holder gets the real view.  Placeholders whose ids are in `last` go behind the others.
        Returns (arena, bytes in front of the first of those)."""
        held = {}
        for holder, attr in fields:
            t = getattr(holder, attr)
            if t is not None and t.device.type == 'meta':
                held.setdefault(id(t), (t, []))[1].append((holder, attr))
        reqs = sorted(held.values(), key=lambda e: id(e[0]) in last)
        offs, total, front = [], 0, None
        for t, _ in reqs:
            if front is None and id(t) in last:
                front = total
            offs.append(total)
            total += _round_up(t.numel() * t.element_size(), 256)
        arena = self._take(name, (max(total, 256),), torch.uint8)
        for (t, holders), off in zip(reqs, offs):
            real = arena[off:off + t.numel() * t.element_size()].view(t.dtype).view(t.shape)
            for holder, attr in holders:
                setattr(holder, attr, real)
        return arena, total if front is None else front

    # ---------------------------------------------------------------------------------------------------------
    def _build(self):
        model, B, dev = self.model, self.B, self.device
        defs, mods = model.module_defs, model.module_list
        n = len(defs)
        shapes = infer_shapes(model, (self.Cin, self.H, self.W),
                              message="layer type '%s' is not supported by the sm_90a training engine yet")
        # a shortcut is folded into the bn+act apply of the conv before it
        lay = build_layout(model, shapes, self.keep_features, lambda i: _block_parts(mods[i])[1] is not None)
        tens, is_head, fused_into = lay.tens, lay.is_head, lay.fused_into
        self.layout = lay
        fo = self.forward_only
        # Activations are bound at their physical widths (layout.phys_width), which are the logical ones on every width
        # the gradient plan accepts.  The rows of a non-head conv's packed forward weights: with a backward, Cout is the
        # K of the data-gradient GEMM and is rounded up to its granule; without one, the output's physical width.
        out_rows = (lambda i: tens[i].Cp) if fo else (lambda i: _round_up(shapes[i][0], 16))
        cidx = lambda i: torch.as_tensor(lay.chmap[i], dtype=torch.long, device=dev)

        # multi-source routes are buffers their producers write into
        for i, parts in lay.concats.items():
            dst = tens[i]
            # a conv reads a placed source through view_k, up to its next 16-channel boundary, which may lie past the
            # concat's own width when a physical width is 8 mod 16 (as in the eval plan)
            wcat = max([dst.Cp] + [off + _round_up(st.Cp, 16) for st, off, placed in parts if placed])
            dst.buf = self._new_buf(('cat', i), wcat, dst.H, dst.W)
            for st, off, placed in parts:
                if placed:
                    st.buf = dst.buf

        def alloc(t, i):
            if t.buf is None:
                t.buf = self._new_buf(('act', i), t.Cp if t.dtype == torch.float16 else head_width(t.C), t.H, t.W,
                                      t.dtype)
            return t

        self.yolo = []
        feat_idx = {}
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            if t == 'se':
                fc = m[0].fc if isinstance(m, nn.Sequential) else m.fc
                src = tens[i - 1]
                out = alloc(tens[i], i)
                cr = fc[0].out_features
                e = _SeRec(i, src, out, fc[0], fc[2], self._take(('se_ws', i), (B, 3 * src.Cp + cr), torch.float32))
                if fo:
                    # fc1 columns / fc2 rows scattered to the input's physical channels (zero for pads and gaps)
                    e.w1 = torch.zeros((cr, src.Cp), dtype=torch.float32, device=dev)
                    e.w2 = torch.zeros((src.Cp, cr), dtype=torch.float32, device=dev)
                    e.cidx = cidx(i - 1)
                self.order.append(('se', e))
                feat_idx[i] = out
            elif t in ('convolutional', 'depthwise'):
                conv, bn, act, slope = _block_parts(m)
                r = _ConvRec()
                r.depthwise = t == 'depthwise'
                if r.depthwise:
                    if conv.groups != conv.in_channels or conv.out_channels != conv.in_channels or bn is None or i == 0:
                        raise NotImplementedError("depthwise block: channel multiplier 1 with BatchNorm expected")
                elif conv.groups != 1:
                    raise NotImplementedError("grouped convolution is not supported by the sm_90a engine yet")
                r.i, r.conv, r.bn, r.act, r.slope = i, conv, bn, act, slope
                r.k, r.s, r.p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
                r.head = is_head[i]
                r.stem = stem_path(conv.in_channels, r.k, None, training=True, batch_norm=bn is not None) \
                    if i == 0 else None
                r.Cout = conv.out_channels
                # GEMM K granules: the output rows of the packed weights, and the forward GEMM's K: the source's physical
                # width up to the MMA K granule (_Tensor.view_k)
                r.Cpad = head_width(r.Cout) if r.head else out_rows(i)
                r.Ipad = _round_up(conv.in_channels if i == 0 else tens[i - 1].Cp, 16)
                if i > 0 and not r.depthwise and lay.chmap[i - 1] != tuple(range(conv.in_channels)):
                    # input columns scattered through the source's channel map.  Shared, not plan-owned: the cached pack
                    # table (keyed by the weight pointers) holds its pointer
                    key = self._tag + (i, lay.chmap[i - 1])
                    if key not in self.shared.col_maps:
                        self.shared.col_maps[key] = torch.as_tensor(lay.chmap[i - 1], dtype=torch.int32, device=dev)
                    r.col_map = self.shared.col_maps[key]
                if r.head and (bn is not None or act != 'linear'):
                    raise NotImplementedError("unsupported YOLO head conv: BatchNorm or a non-linear activation")
                r.src = None if i == 0 else tens[i - 1]
                r.y = alloc(tens[i], i)
                if i + 1 < n and fused_into[i + 1] == i:
                    r.res = tens[sources(i + 1, defs[i + 1]['from'])[0]]
                if bn is not None:
                    if not fo:
                        # csrc/bn_train.cu: a thread owns 8 channels, a CTA of 256 threads at least one pixel row
                        if r.Cout % 8 != 0 or r.Cout > 2048:
                            raise NotImplementedError("layer %d: BatchNorm training needs a multiple of 8 channels, at "
                                                      "most 2048 (got %d)" % (i, r.Cout))
                    # the BatchNorm apply works on the first Cout of Cp channels: a depthwise layer behind a gapped
                    # concat would have its channels elsewhere
                    elif lay.chmap[i] != tuple(range(r.Cout)):
                        raise NotImplementedError("layer %d: BatchNorm over channels a concat placed with gaps" % i)
                    elif r.y.Cp > 2048:
                        raise NotImplementedError("layer %d: BatchNorm of more than 2048 channels (got %d)" % (i, r.Cout))
                    r.z = _Tensor(r.Cout, r.y.H, r.y.W, Cp=r.y.Cp)
                    r.stats = _meta((2, r.y.Cp), torch.float32)
                else:
                    r.z = r.y   # no BN: the conv epilogue applies bias + activation directly
                    r.ones = torch.ones(r.Cpad, dtype=torch.float32, device=dev)
                    r.zeros = torch.zeros(r.Cpad, dtype=torch.float32, device=dev)
                r.aux_row = len(self.convs)
                self.convs.append(r)
                self.order.append(('conv', r))
                if not is_head[i] and r.res is None:
                    feat_idx[i] = r.y   # (a conv with a fused shortcut never materialises its pre-add output)
                if r.depthwise and fo:
                    # fp32 weights scattered to the input's physical channels, re-made by every pack
                    r.wdw = torch.zeros((r.y.Cp,) + tuple(conv.weight.shape[1:]), dtype=torch.float32, device=dev)
                    r.cidx = cidx(i - 1)
            elif t == 'yolo':
                self.yolo.append((m, tens[i - 1]))
            else:
                self.order += pointwise_steps(lay, i, d, m, alloc)
                if t == 'maxpool' and m.__class__.__name__ == 'Sequential':
                    feat_idx[i] = tens[i]
        self.feature_views = [feat_idx.get(i) for i in feature_slots(model)]
        self.feature_maps = [lay.chmap[i] for i in feature_slots(model)]
        # feature_out entries at the logical widths: a slice when the logical channels are the first C physical ones,
        # else (physical view, device index of the logical channels), as the eval plan gives them
        self.fo_features = []
        for t, cmap in zip(self.feature_views, self.feature_maps):
            if t is None:
                self.fo_features.append(None)
            elif cmap[-1] == t.C - 1:
                self.fo_features.append(t.buf[..., t.c0:t.c0 + t.C])
            else:
                self.fo_features.append((t.view(), torch.as_tensor(cmap, device=dev)))
        self.anchors_px = [m.anchors.to(dev).float().contiguous() for (m, _) in self.yolo]
        self.bn_counters = [r.bn.num_batches_tracked for r in self.convs if r.bn is not None]
        # Everything that has to be zero when a pass starts is carved out of ONE allocation per pass, cleared by ONE
        # memset (round 1: one fill launch per buffer, ~450 launches per step).  The forward arena holds the BatchNorm
        # channel sums (sum z, sum z^2) the conv epilogues accumulate into.
        self.fwd_arena, _ = self._carve(('fwd_arena',), [(r, 'stats') for r in self.convs])
        self.params = [p for p in model.parameters()]
        for r in self.convs:
            if not r.stem and not r.depthwise:
                # zero-filled once: the pad rows, the pad / gap columns and the K pad are never written
                key = self._key(r.i)
                if key not in self.shared.w16:
                    self.shared.w16[key] = torch.zeros((r.Cpad, r.k, r.k, r.Ipad), dtype=torch.float16, device=dev)
                r.w16 = self.shared.w16[key]
        # the graph input and the tensor-core stem's im2col workspace (kept for the weight gradient) are taken here, not
        # on first use, so that a larger shape grows every slot while its plan is built
        self.static_x = self._take(('x',), (B, self.Cin, self.H, self.W), torch.float32)
        st = self.convs[0]
        if st.stem == 'im2col':
            d = ops.make_conv_desc((B, self.H, self.W, st.conv.in_channels), st.conv.in_channels, st.y.Cp, st.k, st.s,
                                   st.p, st.y.Cp)
            self.stem_ws = self._take(('stem_ws',), (ops.stem_workspace_bytes(d) // 2,), torch.float16)
        bns = [r for r in self.convs if r.bn is not None]
        if not fo:
            self._build_backward()
        elif bns:
            # without a backward, ONE z slot and one `save` scratch serve every layer: the BatchNorm apply consumes z
            # right after its conv
            zpix = lambda r: B * r.z.H * r.z.W * pitch(r.z.Cp, torch.float16)
            zbuf = self._take(('z',), (max(zpix(r) for r in bns),), torch.float16)
            save = torch.empty(4 * max(r.z.Cp for r in bns), dtype=torch.float32, device=dev)
            for r in bns:
                r.z.buf = zbuf[:zpix(r)].view(B, r.z.H, r.z.W, pitch(r.z.Cp, torch.float16))
                r.save = save[:4 * r.z.Cp].view(4, r.z.Cp)
        self.runs = 0
        self.fwd_graph = self.bwd_graph = None

    def _build_backward(self):
        """The state only a plan with a backward holds: the gradient mirror of the activations, the backward arena, each
        BatchNorm layer's own z and saved statistics, dz, and the data-gradient weight slabs."""
        B, dev, lay = self.B, self.device, self.layout
        for r in self.convs:
            taps = r.conv.in_channels * r.k * r.k
            if r.stem == 'direct' and taps > STEM_WGRAD_MAX_TAPS:
                raise NotImplementedError("layer %d: the weight gradient of a %dx%d first layer on %d channels (%d taps; "
                                          "the direct kernel takes at most %d)" % (r.i, r.k, r.k, r.conv.in_channels,
                                                                                   taps, STEM_WGRAD_MAX_TAPS))
        self.grad_of = {}  # id(_Tensor) -> gradient _Tensor (bf16, same placement)

        def make_grad(t, gbuf, c0=0):
            g = _Tensor(t.C, t.H, t.W, GDT)
            g.buf, g.c0 = gbuf, c0
            self.grad_of[id(t)] = g
            return g

        # the gradients mirror the placement of the multi-source routes and of the grouped ones
        for i, parts in lay.concats.items():
            gdst = make_grad(lay.tens[i], _meta(lay.tens[i].buf.shape, GDT))
            for st, off, placed in parts:
                if placed:
                    make_grad(st, gdst.buf, off)
        for st in self.order:
            t = st[1].y if st[0] in ('conv', 'se') else getattr(st, 'out', None)
            if t is None or id(t) in self.grad_of:
                continue
            if t.dtype == torch.float16:
                make_grad(t, _meta(t.buf.shape, GDT))
            else:  # head output: its gradient is directly the GEMM operand dZ -> fp16 (times a device-side scale)
                hw = head_width(t.C)
                g = self.grad_of[id(t)] = _Tensor(hw, t.H, t.W, torch.float16)
                g.buf = _meta((B, t.H, t.W, hw), torch.float16)
        for i, src in lay.grouped.items():
            gs = self.grad_of[id(src)]
            make_grad(lay.tens[i], gs.buf, gs.c0 + src.C // 2)
        self._plan_grad_writes()

        # The backward arena: activation gradients (bf16; consumers accumulate into them), BN backward sums, the
        # per-layer [max|du|, s, 1/s] scale rows, and the packed fp32 weight gradients (split-K red.add targets)
        self.dz_aux = _meta((len(self.convs) + 1, 4), torch.float32)
        for r in self.convs:
            if r.bn is not None:
                r.sums = _meta((2, r.Cout), torch.float32)
            if r.depthwise:
                r.dwg = _meta(tuple(r.conv.weight.shape), torch.float32)
            elif not r.stem:
                r.dw = _meta((r.Cpad, r.k, r.k, r.Ipad), torch.float32)
        # gradient buffers whose first writer overwrites (see _plan_grad_writes) go behind the part that is memset.  The
        # arena is a slot that plans of other shapes lay out differently, so bytes behind the memset hold whatever the
        # last plan wrote there: a buffer with pad channels (MobileNet widths) stays in the memset part to keep its
        # pad zero.
        width = {}
        for g in self.grad_of.values():
            width[id(g.buf)] = max(width.get(id(g.buf), 0), g.c0 + g.C)
        for g in self.grad_of.values():
            if g.buf.shape[-1] > width[id(g.buf)]:
                self.dirty_grad_bufs.add(id(g.buf))
        clean = {id(g.buf) for g in self.grad_of.values()} - self.dirty_grad_bufs
        self.bwd_arena, self.bwd_zero_bytes = self._carve(
            ('bwd_arena',), [(g, 'buf') for g in self.grad_of.values()] +
            [(r, a) for r in self.convs for a in ('sums', 'dw', 'dwg')] + [(self, 'dz_aux')], clean)
        for st in self.order:
            if st[0] == 'se':
                e = st[1]
                e.ws_bwd = self._take(('se_ws_bwd', e.i), tuple(e.ws.shape), torch.float32)
        # The weight gradients hang off the critical path (dz_i -> dW_i has no consumer until the optimiser), so they run
        # on a second stream concurrently with the data-gradient / BatchNorm chain.  dz is therefore kept per layer
        # (no buffer shared between a running wgrad and the next layer's BN backward).  The pitch is Cout rounded up to
        # the K granule of the data-gradient GEMM; the pad channels stay zero.
        self.dz_bufs = {}
        for r in self.convs:
            if r.bn is not None:
                r.z.buf = self._new_buf(('z', r.i), r.z.Cp, r.z.H, r.z.W)
                # BatchNorm statistics saved by the forward for the backward: [mean, invstd, scale, shift]
                r.save = torch.empty((4, r.Cout), dtype=torch.float32, device=dev)
                full = self._take(('dz', r.i, r.Cpad), (B, r.y.H, r.y.W, r.Cpad), torch.float16)
                self.dz_bufs[r.i] = full[..., :r.Cout]
            if not r.stem and not r.depthwise:
                if r.i not in self.shared.wT:
                    # zero-filled once: the pad rows (>= O) are never written again
                    self.shared.wT[r.i] = torch.zeros(r.Cpad * r.conv.in_channels * r.k * r.k, dtype=torch.float16,
                                                      device=dev)
                r.wT = self.shared.wT[r.i]
        maxc = max(r.Cpad for r in self.convs)
        self.db_scratch = torch.empty(maxc, dtype=torch.float32, device=dev)
        self.stem_dw = torch.empty(maxc * 32, dtype=torch.float32, device=dev)
        self.unpack_table = self.unpack_key = None
        self.bwd_key = None

    # ---------------------------------------------------------------------------------------------------------
    def _params_version(self):
        return sum(p._version for p in self.params)

    def _item_table(self, cls, rows, fields):
        """(device table, items, tiles) of a table-driven launch over the wgmma convolutions (csrc/multi.cu): item j is
        cls(**fields[j]) and starts at the tile after item j - 1's rows[j - 1] / 32 x I / tile_i(k) tiles."""
        from .lib import raw
        items, tiles = [], 0
        for n, f in zip(rows, fields):
            ti = int(raw().b2y_layout_tile_i(f['k']))
            if ti <= 0:
                raise NotImplementedError("kernel size %d is not supported by the training engine" % f['k'])
            items.append(cls(tile_begin=tiles, **f))
            tiles += ((n + 31) // 32) * ((f['I'] + ti - 1) // ti)
        host = torch.frombuffer(bytearray(bytes((cls * len(items))(*items))), dtype=torch.uint8)
        return host.to(self.device), len(items), tiles

    def _pack(self):
        """fp32 master weights -> the operands: ONE table-driven launch over all wgmma convolutions for the fp16 forward
        layout [O][k][k][I] (input columns through the source's channel map) and, with a backward, the per-phase
        data-gradient slabs; the stem's own tiny pack; the forward-only plan's fp32 depthwise / squeeze-excite weights
        scattered to their input's physical channels."""
        from .lib import PackItem
        body = [r for r in self.convs if not r.stem and not r.depthwise]
        key = self._tag + tuple(r.conv.weight.data_ptr() for r in body)
        # one table per set of weight pointers, kept for the life of the shared state: captured graphs of every plan
        # read the table they were captured with
        table = self.shared.pack_tables.get(key)
        if table is None and body:
            for r in body:
                assert r.conv.weight.is_contiguous() and r.conv.weight.dtype == torch.float32
            table = self.shared.pack_tables[key] = self._item_table(PackItem, [r.Cpad for r in body], [dict(
                w=r.conv.weight.data_ptr(), w_fwd=r.w16.data_ptr(), w_dgrad=None if r.wT is None else r.wT.data_ptr(),
                O=r.Cout, Opad=r.Cpad, I=r.conv.in_channels, k=r.k, stride=r.s, pad=r.p, Ipad=r.Ipad,
                col_map=None if r.col_map is None else r.col_map.data_ptr()) for r in body])
        if body:
            tab, n, tiles = table
            call("b2y_pack_conv_weights_multi", ptr(tab), n, tiles, stream_ptr())
        for r in self.convs:
            if r.stem:
                # one row per channel of the output it writes
                r.w32 = _pad_rows(r.conv.weight.detach().float(), self._zview(r).shape[3]).contiguous()
                if r.stem == 'im2col':
                    key = self._key(r.i)
                    if key not in self.shared.wstem:
                        self.shared.wstem[key] = torch.empty((r.w32.shape[0], 32), dtype=torch.float16,
                                                             device=self.device)
                    r.wstem = ops.pack_stem_weights(r.w32, out=self.shared.wstem[key])
            elif r.wdw is not None:
                r.wdw.index_copy_(0, r.cidx, r.conv.weight.detach())
        for st in self.order:
            if st[0] == 'se' and st[1].w1 is not None:
                e = st[1]
                e.w1.index_copy_(1, e.cidx, e.fc1.weight.detach())
                e.w2.index_copy_(0, e.cidx, e.fc2.weight.detach())

    def _plan_grad_writes(self):
        """Which backward write into an activation-gradient buffer is the FIRST one of its channel range.

        Consumers used to accumulate into gradient buffers that the start-of-backward memset had cleared: for yolov4 at
        8 x 640^2 that is ~2.4 GB of memset per step plus a read of zeros by every data-gradient GEMM (another ~2 GB).
        The launch order of the backward pass is static, so the first writer of every (buffer, channel range) is known
        when the plan is built: it OVERWRITES (dgrad accumulate=False, copy instead of add) and the buffer leaves the
        zeroed arena.  A buffer stays 'dirty' (zeroed, accumulate-only) when a first writer cannot overwrite (up-sample /
        max-pool / depthwise / SE backward, stride > kernel dgrad), when ranges overlap partially, or when something would
        read channels nobody has written."""
        self.first_write, cov, dirty = {}, {}, set()
        G = lambda t: self.grad_of[id(t)]

        def write(g, n, key, can_overwrite):
            b, R = id(g.buf), set(range(g.c0, g.c0 + n))
            c = cov.setdefault(b, set())
            inter = R & c
            if not inter and can_overwrite:
                self.first_write[key] = True
            else:
                self.first_write[key] = False
                if inter != R:              # partial overlap, or a first writer that can only accumulate
                    dirty.add(b)
            c |= R

        def read(g, n, c0=None):
            b = id(g.buf)
            c0 = g.c0 if c0 is None else c0
            if not set(range(c0, c0 + n)) <= cov.get(b, set()):
                dirty.add(b)

        for (m, raw) in self.yolo:              # head gradients: written by yolo_grad_to_raw only where a loss exists
            g = G(raw)
            dirty.add(id(g.buf))
            cov[id(g.buf)] = set(range(0, g.C))
        for idx in range(len(self.order) - 1, -1, -1):
            st = self.order[idx]
            kind = st[0]
            if kind == 'conv':
                r = st[1]
                read(G(r.y), G(r.y).C)
                if r.bn is not None and r.res is not None:
                    write(G(r.res), G(r.res).C, ('res', r.i), True)
                if r.stem:
                    continue
                if r.depthwise:
                    write(G(r.src), r.conv.in_channels, ('dwd', r.i), False)
                else:
                    write(G(r.src), r.conv.in_channels, ('dgrad', r.i), r.k >= r.s)
            elif kind == 'se':
                e = st[1]
                read(G(e.y), G(e.y).C)
                write(G(e.src), G(e.src).C, ('se', idx), False)
            elif kind == 'add':
                go = G(st.out)
                read(go, go.C)
                for j, t in enumerate([st.first] + st.others):
                    write(G(t), min(G(t).C, go.C), ('add', idx, j), True)
            elif kind == 'copy':
                gd = G(st.dst)
                read(gd, st.src.C, gd.c0 + st.off)
                write(G(st.src), st.src.C, ('copy', idx), True)
            elif kind in ('upsample', 'maxpool'):
                read(G(st.out), G(st.out).C)
                write(G(st.src), G(st.src).C, (kind, idx), False)
        self.dirty_grad_bufs = dirty

    def _grad_dst(self, param):
        """Where the gradient of `param` is written: its slice of the flat data-parallel buffer (sink), else a
        plan-owned fp32 tensor (handed to autograd as a copy)."""
        if self.sink is not None:
            d = self.sink.get(id(param))
            if d is not None:
                return d
        d = self.shared.own_grads.get(id(param))
        if d is None:
            d = torch.zeros_like(param, dtype=torch.float32, memory_format=torch.contiguous_format)
            self.shared.own_grads[id(param)] = d
        return d

    def _unpack_all(self):
        """packed fp32 weight gradients [O][k][k][I] of all wgmma convolutions -> OIHW destinations, ONE launch."""
        from .lib import UnpackItem
        body = [r for r in self.convs if not r.stem and not r.depthwise]
        dsts = [self._grad_dst(r.conv.weight) for r in body]
        key = tuple(d.data_ptr() for d in dsts)
        if self.unpack_table is None or key != self.unpack_key:
            self.unpack_table = self._item_table(UnpackItem, [r.Cout for r in body], [dict(
                src=r.dw.data_ptr(), dst=d.data_ptr(), O=r.Cout, I=r.conv.in_channels, k=r.k, accumulate=0, Ipad=r.Ipad)
                for r, d in zip(body, dsts)])
            self.unpack_key = key
        tab, n, tiles = self.unpack_table
        call("b2y_unpack_wgrad_multi", ptr(tab), n, tiles, stream_ptr())

    def _zview(self, r):
        return r.z.buf[..., r.z.c0:r.z.c0 + r.Cpad] if r.head else r.z.view()

    # ---- CUDA-graph replay of the two static launch sequences (forward, backward) ------------------------------
    # A training step is ~15 launches per conv layer; issued eagerly from Python the step is CPU-launch bound at 8
    # images per GPU.  Shapes, buffers and the master parameters are static, the per-layer gradient scales live on the
    # device, and the (dynamic) target list only enters the loss between the two graphs.
    def _graphs_enabled(self):
        return getattr(self.model, 'use_cuda_graph', os.environ.get('B2Y_NO_GRAPH', '0') != '1')

    def forward_graphed(self, x):
        if not self._graphs_enabled():
            return self.forward(x)
        if self.runs < 1:                      # first step eager: lazy allocations, warm caches
            self.runs += 1
            return self.forward(x)
        if self.fwd_graph is None:
            self.static_x.copy_(x)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.static_outs = self.forward(self.static_x, force_pack=True)
            self.fwd_graph = g
            self.bwd_graph = None
        self.static_x.copy_(x)
        self.fwd_graph.replay()
        return [o.view_as(o) for o in self.static_outs]

    def backward_graphed(self, dps):
        if not self._graphs_enabled() or self.fwd_graph is None:
            # plan-owned gradient buffers are overwritten by the next step: autograd gets copies
            return {p: g.clone() for p, g in self.backward(dps).items()}
        sink = getattr(self.model, '_b2y_grad_sink', None)
        key = (id(sink), float(getattr(self.model, 'grad_scale', None) or 1.0))
        if self.bwd_graph is None or key != self.bwd_key:
            self.static_dps = [torch.zeros_like(o, dtype=torch.float32) for o in self.static_outs]
            for sd, d in zip(self.static_dps, dps):
                if d is not None:
                    sd.copy_(d)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self.fwd_graph.pool()):
                self.static_grads = self.backward(self.static_dps)
            self.bwd_graph, self.bwd_key = g, key
        for sd, d in zip(self.static_dps, dps):
            if d is None:
                sd.zero_()
            else:
                sd.copy_(d)
        self.bwd_graph.replay()
        # gradients that are not written into a flat sink live in graph-owned memory: hand out copies
        return {p: g.clone() for p, g in self.static_grads.items()}

    def forward(self, x, force_pack=False):
        model = self.model
        ver = self._params_version()
        if force_pack or ver != self.param_version:
            self._pack()
            self.param_version = None if force_pack else ver
        x = x.contiguous().float()
        self.x = x
        self.fwd_arena.zero_()                     # all BatchNorm channel sums (one memset)
        for st in self.order:
            kind = st[0]
            if kind == 'conv':
                r = st[1]
                self._conv_forward(r, x)
            elif kind == 'se':
                e = st[1]
                w1, w2 = (e.fc1.weight.detach(), e.fc2.weight.detach()) if e.w1 is None else (e.w1, e.w2)
                ops.se_fwd(e.src.view(), w1, w2, out=e.y.view(), ws=e.ws)
            else:
                launch_pointwise(st)
        if self.bn_counters:
            torch._foreach_add_(self.bn_counters, 1)

        outs = []
        for (m, raw), anc in zip(self.yolo, self.anchors_px):
            _, p = ops.yolo_decode(raw.buf, m.na, m.no, anc, m.stride, io=None)
            m.nx, m.ny = raw.W, raw.H
            outs.append(p)
        return outs

    def _conv_forward(self, r, x):
        if r.bn is None:
            out = self._zview(r)
            bias = _pad_rows(r.conv.bias.detach() if r.conv.bias is not None else None, out.shape[3])
            if r.stem:
                ops.stem_conv(x, r.w32, bias, r.k, r.s, r.p, act=r.act, slope=r.slope, out=out)
            else:
                ops.conv2d(r.src.view_k(), r.w16, bias, r.k, r.s, r.p, act=r.act, slope=r.slope, out=out)
            return
        z = r.z.view()
        if r.stem == 'im2col':
            # im2col workspace [B*Ho*Wo][32] fp16 (kept for the weight gradient) + one-k-step GEMM with the BN sums
            # coming out of its epilogue
            ops.stem_conv_tc(x, r.wstem, None, r.conv.in_channels, r.k, r.s, r.p, act='linear', out=z,
                             workspace=self.stem_ws, stats=(r.stats[0], r.stats[1]))
        elif r.stem:
            ops.stem_conv(x, r.w32, None, r.k, r.s, r.p, act='linear', out=z)
            # channel sums of the stem output: the reduce kernel with u = z, dy = z gives (sum z, sum z*z)
            if r.ones is None:
                r.ones = torch.ones(z.shape[3], dtype=torch.float32, device=self.device)
                r.zeros = torch.zeros(z.shape[3], dtype=torch.float32, device=self.device)
            B_, H_, W_, C_ = z.shape
            call("b2y_bn_act_bwd_reduce", ptr(z), ops._pitch(z), ptr(z), ops._pitch(z), ptr(r.ones), ptr(r.zeros),
                 ptr(r.zeros), ptr(r.ones), ptr(r.stats[1]), ptr(r.stats[0]), None, B_ * H_ * W_, C_, 0, 0.0, 0,
                 stream_ptr())
        elif r.depthwise:
            w = r.conv.weight.detach() if r.wdw is None else r.wdw
            ops.dwconv2d(r.src.view(), w, r.k, r.s, r.p, out=z, stats=(r.stats[0], r.stats[1]))
        else:
            ops.conv2d(r.src.view_k(), r.w16[:z.shape[3]], None, r.k, r.s, r.p, out=z, stats=(r.stats[0], r.stats[1]))
        bn = r.bn
        count = z.shape[0] * z.shape[1] * z.shape[2]
        res = r.res.view() if r.res is not None else None
        y = r.y.view()
        # z, y and the statistics are Cp wide; gamma, beta and the running statistics are the module's own Cout
        call("b2y_bn_train_fwd_lw", ptr(z), ops._pitch(z), ptr(r.stats[0]), ptr(r.stats[1]), int(count),
             ptr(bn.weight.detach()), ptr(bn.bias.detach()), float(bn.eps), float(bn.momentum),
             ptr(bn.running_mean), ptr(bn.running_var), ptr(r.save), ptr(res),
             ops._pitch(res) if res is not None else 0, ptr(y), ops._pitch(y), int(count), z.shape[3], r.Cout,
             ACT[r.act], float(r.slope), stream_ptr())

    # ---------------------------------------------------------------------------------------------------------
    def backward(self, dps):
        """dps: gradients w.r.t. the yolo outputs p (fp32). Returns {param: grad} for every model parameter."""
        # gradients flow in bf16, so no loss scaling is needed; model.grad_scale (power of two) is still honoured
        S = float(getattr(self.model, 'grad_scale', None) or 1.0)
        self.last_grad_scale = S
        inv = 1.0 / S
        self.sink = getattr(self.model, '_b2y_grad_sink', None)   # FlatDataParallel: write into the flat buffer
        # one memset: BN sums, scale rows, packed weight gradients and the activation gradients that are accumulate-only
        self.bwd_arena[:max(self.bwd_zero_bytes, 1)].zero_()
        if self.shared.side_stream is None:
            self.shared.side_stream = torch.cuda.Stream(device=self.device)
        self.side_stream = self.shared.side_stream
        grads = {}
        # head gradients are GEMM operands (fp16): scale them by a power of two derived on the device from max|dp|
        live = [dp for dp in dps if dp is not None]
        amax = torch.stack([dp.detach().abs().max() for dp in live]).max().clamp(min=1e-30)
        # 2^floor(log2(4096 / amax)) = the value with its mantissa bits cleared (no exp2 / log2: torch compiles those
        # through NVRTC on first use, which every rank of a multi-GPU job would do at the same moment)
        hs = ((4096.0 / amax).float().view(torch.int32) & 0x7F800000).view(torch.float32).clamp(1e-30, 1e30)
        self.head_scale = torch.stack([hs, 1.0 / hs]).contiguous()           # device [s, 1/s]
        for (m, raw), dp in zip(self.yolo, dps):
            g = self.grad_of[id(raw)]
            if dp is None:
                continue
            call("b2y_yolo_grad_to_raw", ptr(dp.contiguous().float()), ptr(g.buf), g.C, self.B, m.na, m.no, raw.H,
                 raw.W, S, ptr(self.head_scale), ops._gdt(g.buf), stream_ptr())
        G = lambda t: self.grad_of[id(t)]
        for idx in range(len(self.order) - 1, -1, -1):
            st = self.order[idx]
            kind = st[0]
            if kind == 'conv':
                self._conv_backward(st[1], grads, S, inv)
            elif kind == 'se':
                e = st[1]
                ops.se_bwd(e.src.view(), G(e.y).view(), e.fc1.weight.detach(), e.fc2.weight.detach(), e.ws,
                           G(e.src).view(), accumulate=True, dw1=self._grad_dst(e.fc1.weight),
                           dw2=self._grad_dst(e.fc2.weight), grad_scale=inv, ws_bwd=e.ws_bwd)
            elif kind == 'add':
                go = G(st.out).view()
                for j, s in enumerate([st.first] + st.others):
                    gs = G(s).view()
                    n = min(gs.shape[3], go.shape[3])      # sliced addends receive the matching gradient channels
                    if self.first_write.get(('add', idx, j)):
                        ops.copy_channels(go[..., :n], gs[..., :n])
                    else:
                        ops.add(gs[..., :n], go[..., :n], out=gs[..., :n])
            elif kind == 'copy':
                gd = G(st.dst)
                gs = G(st.src).view()
                gslice = gd.buf[..., gd.c0 + st.off:gd.c0 + st.off + st.src.C]
                if self.first_write.get(('copy', idx)):
                    ops.copy_channels(gslice, gs)
                else:
                    ops.add(gs, gslice, out=gs)
            elif kind == 'upsample':
                src = st.src
                gy, gx = G(st.out).view(), G(src).view()
                call("b2y_upsample_nearest_bwd", ptr(gy), ops._pitch(gy), ptr(gx), ops._pitch(gx), self.B, src.H,
                     src.W, src.C, int(st.stride), ops._gdt(gy), stream_ptr())
            elif kind == 'maxpool':
                src = st.src
                gy, gx, xv = G(st.out).view(), G(src).view(), src.view()
                call("b2y_maxpool_bwd", ptr(xv), ops._pitch(xv), ptr(gy), ops._pitch(gy), ptr(gx), ops._pitch(gx),
                     self.B, src.H, src.W, src.C, int(st.k), int(st.s), 1 if st.tiny_pad else 0, ops._gdt(gy),
                     stream_ptr())
        torch.cuda.current_stream().wait_stream(self.side_stream)          # join: every weight gradient is complete
        self._unpack_all()
        if self.shared.own_grads:
            # plain-autograd path: hand out copies (the shared buffers are overwritten by the next step)
            by_id = {id(p): p for p in self.params}
            for pid, g in self.shared.own_grads.items():
                grads[by_id[pid]] = g
        return grads

    def _conv_backward(self, r, grads, S, inv):
        B = self.B
        gy = self.grad_of[id(r.y)]
        conv, bn = r.conv, r.bn
        Ho, Wo = r.y.H, r.y.W
        if bn is not None:
            dy = gy.view()
            if r.res is not None:   # fused shortcut: the same gradient also flows to the skip source
                gs = self.grad_of[id(r.res)].view()
                if self.first_write.get(('res', r.i)):
                    ops.copy_channels(dy, gs)
                else:
                    ops.add(gs, dy, out=gs)
            dz = self.dz_bufs[r.i]
            aux = self.dz_aux[r.aux_row]
            inv_s = aux[2:3]                                   # device scalar 1/s of this layer's dz
            z = r.z.view()
            pixels = B * Ho * Wo
            a = ACT[r.act]
            call("b2y_bn_train_bwd_reduce", ptr(z), ops._pitch(z), ptr(dy), ops._pitch(dy), ptr(r.save),
                 ptr(r.sums), ptr(aux), pixels, r.Cout, a, float(r.slope), ops._gdt(dy), stream_ptr())
            call("b2y_bn_train_bwd_apply", ptr(z), ops._pitch(z), ptr(dy), ops._pitch(dy),
                 ptr(bn.weight.detach()), ptr(r.save), ptr(r.sums), ptr(dz), ops._pitch(dz), pixels, r.Cout, a,
                 float(r.slope), ops._gdt(dy), ptr(aux), C.c_void_p(aux.data_ptr() + 4),
                 ptr(self._grad_dst(bn.weight)), ptr(self._grad_dst(bn.bias)), float(inv), stream_ptr())
        else:
            dz = gy.buf[..., :r.Cpad] if r.head else gy.view()
            inv_s = self.head_scale[1:2]
            if r.act != 'linear':
                raise NotImplementedError("activation without BatchNorm in training")
            if conv.bias is not None:
                db = self.db_scratch[:r.Cpad]
                db.zero_()
                ops.bias_act_bwd_reduce(dz, dz, r.ones, r.zeros, 'linear', dbeta=db)
                self._emit(grads, conv.bias, db[:r.Cout] * inv_s, inv)
        I = conv.in_channels
        if r.stem == 'im2col':
            # dW = dz^T . im2col(x): the pixel-dimension GEMM on the tensor cores over the forward's workspace
            gw = self._grad_dst(conv.weight)
            kk = I * r.k * r.k
            xcol = self.stem_ws[:B * Ho * Wo * 32].view(B, Ho, Wo, 32)
            dwp = self.stem_dw[:r.Cpad * 32].view(r.Cpad, 1, 1, 32)
            dwp.zero_()
            ops.conv2d_bwd_weight(xcol, dz, 1, 1, 0, scale=inv, dw=dwp, inv_scale=inv_s)
            gw.copy_(dwp[:r.Cout, 0, 0, :kk].view(r.Cout, r.k, r.k, I).permute(0, 3, 1, 2))
        elif r.stem:
            gw = self._grad_dst(conv.weight)
            gw.zero_()
            d = ConvDesc(B, self.H, self.W, I, I, r.Cout, r.k, r.s, r.p, Ho, Wo, ops._pitch(dz), 0, 0.0, OUT_F16, 0)
            call("b2y_stem_conv_bwd_weight", C.byref(d), ptr(self.x), ptr(dz), ptr(gw), inv, ops._gdt(dz), stream_ptr())
            gw.mul_(inv_s)
        elif r.depthwise:
            xs = r.src.view()
            ops.dwconv2d_bwd_weight(xs, dz, r.k, r.s, r.p, alpha=inv, dw=r.dwg, inv_scale=inv_s)
            ops.axpby(r.dwg.reshape(-1), self._grad_dst(conv.weight).reshape(-1), 1.0, 0.0)
            gx = self.grad_of[id(r.src)]
            ops.dwconv2d_bwd_data(dz, conv.weight.detach(), (B, r.src.H, r.src.W, I), r.k, r.s, r.p, out=gx.view(),
                                  accumulate=True, inv_scale=inv_s)
        else:
            # packed fp32 gradient slice (zeroed with the backward arena); unpacked for all layers at the end.
            # K operands are taken with their zero pad: x with Ipad channels, dz with Cpad channels.
            xk = r.src.view_k()
            dzk = dz if dz.shape[3] == r.Cpad else _widen(dz, r.Cpad)
            self.side_stream.wait_stream(torch.cuda.current_stream())   # dz (and 1/s) of this layer are complete
            with torch.cuda.stream(self.side_stream):
                ops.conv2d_bwd_weight(xk, dzk, r.k, r.s, r.p, scale=inv, dw=r.dw, inv_scale=inv_s)
            gx = self.grad_of[id(r.src)]
            ops.conv2d_bwd_data(dzk, r.wT, (B, r.src.H, r.src.W, I), r.k, r.s, r.p, out=gx.view(),
                                accumulate=not self.first_write.get(('dgrad', r.i), False), inv_scale=inv_s)

    def _emit(self, grads, param, src, alpha):
        ops.axpby(src.contiguous(), self._grad_dst(param), alpha, 0.0)

    # ---------------------------------------------------------------------------------------------------------
    def run(self, x):
        """autograd entry: returns (yolo_out list, feature_out at the logical widths).  While the step's backward is
        pending (autograd recorded it), the plan's slot store is pinned: the engine runs plans of other shapes on private
        storage."""
        if self.forward_only:
            with torch.no_grad():
                outs = self.forward_graphed(x)
        else:
            outs = _DarknetTrain.apply(self, x, *self.params)
            if outs[0].grad_fn is not None:
                outs[0].grad_fn.b2y_pin = _Pin(self.store, self)   # released by backward or when the graph is freed
        # the running statistics were just updated through raw pointers (also under graph replay): eval plans re-fold
        object.__setattr__(self.model, '_b2y_epoch', getattr(self.model, '_b2y_epoch', 0) + 1)
        return list(outs), LazyFeatures(self.fo_features)


class _DarknetTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, plan, x, *params):
        ctx.plan = plan
        ctx.params = params
        with torch.no_grad():
            outs = plan.forward_graphed(x)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *dps):
        plan = ctx.plan
        with torch.no_grad():
            grads = plan.backward_graphed(dps)
        pin = getattr(ctx, 'b2y_pin', None)
        if pin is not None:
            pin.release()
        out = []
        for p in ctx.params:
            g = grads.get(p)
            out.append(g if (g is not None and p.requires_grad) else None)
        return (None, None) + tuple(out)
