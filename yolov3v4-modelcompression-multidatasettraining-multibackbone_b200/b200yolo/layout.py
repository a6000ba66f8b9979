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


def pitch(C, dtype):
    """Channel pitch of a buffer that holds C channels: fp16 activations are padded to the MMA K granule (16 elements;
    the pad channels are zero and nobody writes them), everything else to 4."""
    g = 16 if dtype == torch.float16 else 4
    return (C + g - 1) // g * g


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
                tensor's buffer"""
    __slots__ = ('shapes', 'is_head', 'fused_into', 'tens', 'concats', 'grouped')


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
        if d['type'] == 'shortcut' and i > 1:
            frm = sources(i, d['from'])
            if (not keep_features  # feature_out must expose the conv output *before* the add
                    and len(frm) == 1 and defs[i - 1]['type'] == 'convolutional' and not routs[i - 1]
                    and not getattr(mods[i], 'weight', False) and shapes[frm[0]] == shapes[i - 1] and fuse_ok(i - 1)):
                fused_into[i] = i - 1

    is_alias = lambda d: d['type'] == 'route' and len(d['layers']) == 1 and 'groups' not in d
    tens = lay.tens = [None] * n
    for i, d in enumerate(defs):
        if d['type'] != 'yolo' and not is_alias(d):
            tens[i] = _Tensor(*shapes[i], torch.float32 if is_head[i] else torch.float16)
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

    # concat placement: a source is written in place when it is fp16, not yet inside another concat, not a concat
    # itself, and starts on a 16-byte boundary of the pixel row; otherwise it is copied
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
            off += st.C
        lay.concats[i] = parts
    lay.grouped = {}
    for i, d in enumerate(defs):
        if d['type'] == 'route' and len(d['layers']) == 1 and 'groups' in d:
            src = tens[i - 1]
            tens[i].c0 = src.c0 + src.C // 2
            lay.grouped[i] = src
    return lay
