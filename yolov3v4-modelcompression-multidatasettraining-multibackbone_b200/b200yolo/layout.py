"""How a Darknet cfg becomes activation tensors: the one place that reads `module_defs` for shapes and placement.

The inference plan (engine.py), the training plan (train_engine.py) and the INT8 plan (qengine.py) all need the
(C, H, W) of every layer; the first two also share which shortcuts are folded into the conv before them, which routes
are aliases, and the zero-copy concat placement (route/concat producers write straight into their channel slot of the
concat buffer).  This module decides all of that from the model alone: no device, no kernels, no allocation.  A plan
binds `_Tensor.buf` when it allocates, with its own slot names and dtypes.
"""
import torch
import torch.nn as nn

_ACT_OF_CLASS = {'LeakyReLU': 'leaky', 'Mish': 'mish', 'ReLU6': 'relu6', 'HardSwish': 'h_swish', 'ReLU': 'relu',
                 'Swish': 'swish'}
LAYER_TYPES = ('convolutional', 'depthwise', 'se', 'maxpool', 'upsample', 'route', 'shortcut', 'yolo')


def phys_width(C):
    """Physical channel count of an fp16 activation with C logical channels: whole 8-channel groups (16 bytes), which
    every elementwise, depthwise and squeeze-excite kernel and the 16-byte alignment of concat slots need.  Channels
    C .. phys_width(C) - 1 hold zeros (see Layout.chmap)."""
    return (C + 7) // 8 * 8


class _Tensor:
    """Activation tensor of C logical channels stored as Cp physical ones: NHWC view = buffer[..., c0:c0+Cp]."""
    __slots__ = ('C', 'Cp', 'H', 'W', 'buf', 'c0', 'dtype')

    def __init__(self, C, H, W, dtype=torch.float16, Cp=None):
        self.C, self.H, self.W, self.dtype = C, H, W, dtype
        self.Cp = C if Cp is None else Cp
        self.buf, self.c0 = None, 0

    def view(self):
        return self.buf[..., self.c0:self.c0 + self.Cp]

    def view_k(self):
        """View for a tensor-core consumer: the channel count rounded up to 16 (the MMA K granule is 16 fp16 elements).
        MobileNet widths (24, 40, 72, 120, 184, 200) are not: their buffers are allocated zero-filled with a pitch that
        is a multiple of 16 and nobody ever writes the pad channels, the packed weights carry zero columns there (a
        tensor living inside a concat buffer may see its neighbour's channels instead of zeros: finite values times
        zero weights)."""
        ck = (self.Cp + 15) // 16 * 16
        if ck == self.Cp:
            return self.view()
        if self.c0 + ck > self.buf.shape[3]:
            raise RuntimeError("activation buffer too narrow for the padded channel view (C=%d)" % self.Cp)
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


def pitch(C, dtype):
    """Channel pitch of a buffer that holds C channels: fp16 activations are padded to the MMA K granule (16 elements;
    the pad channels are zero and nobody writes them), everything else to 4."""
    g = 16 if dtype == torch.float16 else 4
    return (C + g - 1) // g * g


STEM_WGRAD_MAX_TAPS = 40    # b2y_stem_conv_bwd_weight: 8 tap groups of 5 taps per output channel


def stem_path(in_c, k, out_c, training=False, batch_norm=True):
    """Kernel path of the first convolution, which reads the NCHW image (include/b200yolo.h, b2y_pack_stem_weights).

    'fused'   b2y_stem_conv_fwd_fused: the im2col tile built in shared memory, inference with out_c <= 64
    'im2col'  b2y_stem_conv_fwd_tc: the im2col matrix written to a workspace, then one GEMM, for wider inference
              outputs; in training its epilogue gives the BatchNorm batch sums and the workspace feeds the weight
              gradient, so a stem without BatchNorm (bias and activation in the direct kernel) stays direct
    'direct'  b2y_stem_conv_fwd (and b2y_stem_conv_bwd_weight) on CUDA cores, any k

    The two im2col kernels are compiled for the (in_c, k) pairs with odd k and in_c * k * k <= 32 (one output pixel's
    receptive field fits one 32-column fp16 GEMM row), the list B2Y_STEM_IM2COL_SHAPES of csrc/common.cuh.  out_c is
    the width the stem writes (its physical width in the plans)."""
    if in_c > 4:
        raise NotImplementedError("first layer with more than 4 input channels")
    if k % 2 == 0 or in_c * k * k > 32:
        return 'direct'
    if training:
        return 'im2col' if batch_norm else 'direct'
    return 'fused' if out_c <= 64 else 'im2col'


def pair_form(k, s, p, cin, cout, in_w):
    """Pixel-pair form of a non-stem convolution, the one shape rule of the fp16 and INT8 eval plans (why the pairs pay:
    engine.Plan._pair_pack).  The NHWC input [B,H,W,32] is read as pixel pairs [B,H,W/2,64]:

    's1'  3x3 stride 1, cout <= 128 and a multiple of 8: a 3x3 conv over the pairs with 64 input and 2 * cout output
          channels (ops.s1_pair_weights), its output read as pairs too
    's2'  3x3 stride 2: B2Y_WLAYOUT_S2_PAIRS, a 3 x 2 window with stride 2 x 1 over the pairs (ops.s2_pair_weights)
    None  the dense form

    A plan may add conditions on where its tensors are placed."""
    if k != 3 or p != 1 or cin != 32 or in_w % 2:
        return None
    if s == 1 and cout <= 128 and cout % 8 == 0:
        return 's1'
    return 's2' if s == 2 else None


def sources(i, rel):
    """Absolute layer indices of the `layers=` / `from=` list of layer i (negative entries are relative to i)."""
    return [i + l if l < 0 else l for l in rel]


def feature_slots(model):
    """Layers that have an entry in feature_out (reference models.py:542-543): every nn.Sequential block whose
    successor is not a YOLO layer."""
    defs = model.module_defs
    return [i for i, m in enumerate(model.module_list)
            if m.__class__.__name__ == 'Sequential' and i + 1 < len(defs) and defs[i + 1]['type'] != 'yolo']


def infer_shapes(model, chw, supported=LAYER_TYPES, message="layer type '%s' is not supported by the sm_90a engine yet"):
    """(C, H, W) of every layer's output for an input of chw = (C, H, W)."""
    shapes, prev = [], tuple(chw)
    for i, (d, m) in enumerate(zip(model.module_defs, model.module_list)):
        t = d['type']
        if t not in supported:
            raise NotImplementedError(message % t)
        C, H, W = prev
        if t in ('convolutional', 'depthwise'):
            conv = _block_parts(m)[0]
            k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
            H, W = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
            C = conv.out_channels
        elif t == 'maxpool':
            k, s = d['size'], d['stride']
            if k == 2 and s == 1:       # yolov3-tiny: zero-padded on the right / bottom only, the size is kept
                H, W = (H + 1 - k) // s + 1, (W + 1 - k) // s + 1
            else:
                p = (k - 1) // 2
                H, W = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        elif t == 'upsample':
            H, W = H * d['stride'], W * d['stride']
        elif t == 'route':
            srcs = sources(i, d['layers'])
            C = sum(shapes[s][0] for s in srcs)
            if 'groups' in d:
                C //= 2
            H, W = shapes[srcs[0]][1], shapes[srcs[0]][2]
        prev = (C, H, W)
        shapes.append(prev)
    return shapes


class Layout:
    """shapes      (C, H, W) per layer
    is_head     conv directly followed by a yolo layer: fp32 output
    fused_into  shortcut i is folded into conv fused_into[i] (= i - 1), which writes the shortcut's tensor
    tens        the _Tensor of every layer (None for yolo layers); single-source routes share their source's tensor,
                a conv with a fused shortcut shares the shortcut's
    concats     {multi-source route i: [(source tensor, channel offset, placed)]}: a placed source lives inside the
                route's buffer (its c0 is the offset, the plan gives it the route's buffer), the others are copied
    grouped     {grouped route i: the tensor whose upper channel half it is}; its c0 is set, the plan gives it that
                tensor's buffer
    chmap       per layer (None for yolo layers): the physical channel, relative to the tensor's c0, of each logical
                channel.  The identity except behind a multi-source route, whose sources sit at offsets that are sums
                of physical widths, with zero channels between them; every layer that works channel by channel
                (depthwise, squeeze-excite, max-pool, up-sample, shortcut) keeps its input's map.  A consumer of weights
                scatters its input columns through it."""
    __slots__ = ('shapes', 'is_head', 'fused_into', 'tens', 'concats', 'grouped', 'chmap')


def _channel_maps(defs, shapes, is_head):
    """(physical width, logical -> physical channel map) of every layer's output tensor, in layer order."""
    n = len(defs)
    cp, chmap = [None] * n, [None] * n
    for i, d in enumerate(defs):
        t, C = d['type'], shapes[i][0]
        if t == 'yolo':
            continue
        if t == 'convolutional':
            cp[i], chmap[i] = (C if is_head[i] else phys_width(C)), tuple(range(C))
        elif t in ('depthwise', 'se', 'maxpool', 'upsample'):
            cp[i], chmap[i] = cp[i - 1], chmap[i - 1]
        elif t == 'shortcut':
            cp[i], chmap[i] = cp[i - 1], chmap[i - 1]
            for s in sources(i, d['from']):
                k = min(C, shapes[s][0])
                if chmap[s][:k] != chmap[i - 1][:k]:
                    raise NotImplementedError("layer %d: shortcut over addends whose channels are placed differently "
                                              "(one of them is a concat of widths that are not multiples of 8)" % i)
                if shapes[s][0] > C and min(cp[s], cp[i]) > C:
                    # the add covers whole 8-channel groups and would write the wider addend into the pad channels
                    raise NotImplementedError("layer %d: shortcut whose addend is wider than its %d-channel input, "
                                              "which is not a multiple of 8" % (i, C))
        elif t == 'route':
            srcs = sources(i, d['layers'])
            if len(srcs) > 1:
                off, m = 0, []
                for s in srcs:
                    m += [off + c for c in chmap[s]]
                    off += cp[s]
                cp[i], chmap[i] = off, tuple(m)
            elif 'groups' in d:
                src_map = chmap[i - 1]
                half = len(src_map) // 2
                p0 = src_map[half]
                if len(src_map) % 2 or p0 % 8:
                    raise NotImplementedError("layer %d: grouped route over %d channels: its upper half does not start "
                                              "on an 8-channel boundary" % (i, len(src_map)))
                cp[i], chmap[i] = cp[i - 1] - p0, tuple(c - p0 for c in src_map[half:])
            else:
                cp[i], chmap[i] = cp[srcs[0]], chmap[srcs[0]]
    return cp, chmap


def build_layout(model, shapes, keep_features, fuse_ok):
    """fuse_ok(i): the mode-specific part of "conv i can take the shortcut that follows it" (inference: a channel count
    the residual epilogue can read; training: a BatchNorm, whose apply kernel does the add)."""
    defs, mods, routs = model.module_defs, model.module_list, model.routs
    n = len(defs)
    lay = Layout()
    lay.shapes = shapes
    is_head = lay.is_head = [False] * n
    fused_into = lay.fused_into = [None] * n
    for i, d in enumerate(defs):
        if d['type'] == 'yolo' and i > 0 and defs[i - 1]['type'] == 'convolutional':
            is_head[i - 1] = True
    cp, chmap = _channel_maps(defs, shapes, is_head)
    lay.chmap = chmap
    for i, d in enumerate(defs):
        if d['type'] == 'shortcut' and i > 1:
            frm = sources(i, d['from'])
            if (not keep_features  # feature_out must expose the conv output *before* the add
                    and len(frm) == 1 and defs[i - 1]['type'] == 'convolutional' and not routs[i - 1]
                    and not getattr(mods[i], 'weight', False) and shapes[frm[0]] == shapes[i - 1]
                    and chmap[frm[0]] == chmap[i - 1] and cp[frm[0]] == cp[i - 1] and fuse_ok(i - 1)):
                fused_into[i] = i - 1

    is_alias = lambda d: d['type'] == 'route' and len(d['layers']) == 1 and 'groups' not in d
    tens = lay.tens = [None] * n
    for i, d in enumerate(defs):
        if d['type'] != 'yolo' and not is_alias(d):
            tens[i] = _Tensor(*shapes[i], torch.float32 if is_head[i] else torch.float16, Cp=cp[i])
    for i in range(n):
        if fused_into[i] is not None:
            tens[fused_into[i]] = tens[i]
    alias = {}
    for i, d in enumerate(defs):
        if is_alias(d):
            src = sources(i, d['layers'])[0]
            while src in alias:
                src = alias[src]
            alias[i] = src
            tens[i] = tens[src]

    # concat placement at physical offsets: a source is written in place when it is fp16, not yet inside another
    # concat, not a concat itself, and starts on a 16-byte boundary of the pixel row; otherwise it is copied
    lay.concats = {}
    taken = set()
    for i, d in enumerate(defs):
        if d['type'] != 'route' or len(d['layers']) == 1:
            continue
        dst = tens[i]
        taken.add(id(dst))
        parts, off = [], 0
        for s in sources(i, d['layers']):
            st = tens[s]
            placed = id(st) not in taken and off % 8 == 0 and st.dtype == torch.float16
            if placed:
                st.c0 = off
                taken.add(id(st))
            parts.append((st, off, placed))
            off += st.Cp
        lay.concats[i] = parts
    lay.grouped = {}
    for i, d in enumerate(defs):
        if d['type'] == 'route' and len(d['layers']) == 1 and 'groups' in d:
            src = tens[i - 1]
            tens[i].c0 = src.c0 + src.Cp - tens[i].Cp
            lay.grouped[i] = src
    return lay
