"""Programmatic Darknet .cfg generator for the benchmark architectures.

The reference ships its cfg files under cfg/**; they are data, not code, and are not copied into this repo.
This module re-creates the architectures (YOLOv3 / Darknet-53, YOLOv3-tiny, YOLOv4 / CSPDarknet-53 + SPP + PAN,
YOLOv4-tiny, YOLOv2 / Darknet-19 and YOLOv2-tiny with one 5-anchor head, the MobileNetV3 and GhostNet backbones under a
YOLOv3 head) from their published structure so that tests and bench.py work on a box without /root/reference.
tests/test_cfg_parity.py checks (when the reference is present) that the generated text parses to the same
module definitions as the reference's own cfg files.
"""

COCO_ANCHORS_V3 = "10,13, 16,30, 33,23, 30,61, 62,45, 59,119, 116,90, 156,198, 373,326"
COCO_ANCHORS_V4 = "12, 16, 19, 36, 40, 28, 36, 75, 76, 55, 72, 146, 142, 110, 192, 243, 459, 401"
TINY_ANCHORS = "10,14, 23,27, 37,58, 81,82, 135,169, 344,319"
V2_ANCHORS = "7,12, 19,30, 45,61, 90,141, 240,279"


class _Cfg:
    def __init__(self, net):
        self.lines = ["[net]"] + ["%s=%s" % kv for kv in net] + [""]
        self.n = 0  # number of layers emitted so far

    def block(self, kind, *kvs):
        self.lines.append("[%s]" % kind)
        self.lines += ["%s=%s" % kv for kv in kvs]
        self.lines.append("")
        self.n += 1
        return self.n - 1

    def conv(self, filters, size, stride=1, act="leaky", bn=1):
        kv = ([("batch_normalize", 1)] if bn else []) + [("filters", filters), ("size", size), ("stride", stride),
                                                         ("pad", 1), ("activation", act)]
        return self.block("convolutional", *kv)

    def depthwise(self, filters, size, stride=1, act="relu6"):
        return self.block("depthwise", ("batch_normalize", 1), ("filters", filters), ("size", size), ("stride", stride),
                          ("pad", 1), ("activation", act))

    def se(self, filters):
        return self.block("se", ("filters", filters))

    def shortcut(self, frm=-3):
        return self.block("shortcut", ("from", frm), ("activation", "linear"))

    def route(self, *layers):
        return self.block("route", ("layers", ",".join(str(l) for l in layers)))

    def upsample(self, s=2):
        return self.block("upsample", ("stride", s))

    def maxpool(self, size, stride):
        return self.block("maxpool", ("stride", stride), ("size", size))

    def yolo(self, mask, anchors, classes, num, extra=()):
        return self.block("yolo", ("mask", ",".join(str(m) for m in mask)), ("anchors", anchors),
                          ("classes", classes), ("num", num), ("jitter", ".3"), ("ignore_thresh", ".7"),
                          ("truth_thresh", 1), *extra)

    def text(self):
        return "\n".join(self.lines)


def _net(width=416, height=416, momentum="0.9"):
    return [("batch", 64), ("subdivisions", 16), ("width", width), ("height", height), ("channels", 3),
            ("momentum", momentum), ("decay", "0.0005"), ("angle", 0), ("saturation", "1.5"), ("exposure", "1.5"),
            ("hue", ".1"), ("learning_rate", "0.001"), ("burn_in", 1000), ("max_batches", 500200),
            ("policy", "steps"), ("steps", "400000,450000"), ("scales", ".1,.1")]


def yolov3(classes=80):
    c = _Cfg(_net())
    nout = 3 * (classes + 5)
    c.conv(32, 3)
    for filters, blocks in ((64, 1), (128, 2), (256, 8), (512, 8), (1024, 4)):
        c.conv(filters, 3, 2)
        for _ in range(blocks):
            c.conv(filters // 2, 1)
            c.conv(filters, 3)
            c.shortcut(-3)
    # detection head, three scales (strides 32, 16, 8)
    for scale, (mid, mask, skip) in enumerate(((512, (6, 7, 8), None), (256, (3, 4, 5), 61), (128, (0, 1, 2), 36))):
        if skip is not None:
            c.route(-4)
            c.conv(mid, 1)
            c.upsample(2)
            c.route(-1, skip)
        for _ in range(3):
            c.conv(mid, 1)
            c.conv(mid * 2, 3)
        c.conv(nout, 1, act="linear", bn=0)
        c.yolo(mask, COCO_ANCHORS_V3, classes, 9, (("random", 1),))
    return c.text()


def yolov3_tiny(classes=80):
    c = _Cfg(_net())
    nout = 3 * (classes + 5)
    for i, f in enumerate((16, 32, 64, 128, 256, 512)):
        c.conv(f, 3)
        c.maxpool(2, 2 if i < 5 else 1)
    c.conv(1024, 3)
    c.conv(256, 1)
    c.conv(512, 3)
    c.conv(nout, 1, act="linear", bn=0)
    c.yolo((3, 4, 5), TINY_ANCHORS, classes, 6, (("random", 1),))
    c.route(-4)
    c.conv(128, 1)
    c.upsample(2)
    c.route(-1, 8)
    c.conv(256, 3)
    c.conv(nout, 1, act="linear", bn=0)
    c.yolo((0, 1, 2), TINY_ANCHORS, classes, 6, (("random", 1),))
    return c.text()


def _csp_stage(c, filters, blocks, first=False):
    """One CSPDarknet stage: stride-2 conv, split into two 1x1 branches, `blocks` residual units, merge."""
    half = filters if first else filters // 2
    c.conv(filters, 3, 2, act="mish")
    c.conv(half, 1, act="mish")          # shortcut branch
    c.route(-2)
    c.conv(half, 1, act="mish")          # main branch
    for _ in range(blocks):
        c.conv(filters // 2, 1, act="mish")
        c.conv(half, 3, act="mish")
        c.shortcut(-3)
    c.conv(half, 1, act="mish")
    c.route(-1, -(3 * blocks + 4))
    c.conv(filters, 1, act="mish")


def yolov4(classes=80):
    c = _Cfg(_net(608, 608, "0.949"))
    nout = 3 * (classes + 5)
    c.conv(32, 3, act="mish")
    _csp_stage(c, 64, 1, first=True)
    _csp_stage(c, 128, 2)
    _csp_stage(c, 256, 8)     # ends at layer 54
    _csp_stage(c, 512, 8)     # ends at layer 85
    _csp_stage(c, 1024, 4)    # ends at layer 104
    # SPP neck
    c.conv(512, 1)
    c.conv(1024, 3)
    c.conv(512, 1)
    c.maxpool(5, 1)
    c.route(-2)
    c.maxpool(9, 1)
    c.route(-4)
    c.maxpool(13, 1)
    c.route(-1, -3, -5, -6)
    c.conv(512, 1)
    c.conv(1024, 3)
    c.conv(512, 1)
    # PAN top-down
    for mid, lateral in ((256, 85), (128, 54)):
        c.conv(mid, 1)
        c.upsample(2)
        c.route(lateral)
        c.conv(mid, 1)
        c.route(-1, -3)
        c.conv(mid, 1)
        c.conv(mid * 2, 3)
        c.conv(mid, 1)
        c.conv(mid * 2, 3)
        c.conv(mid, 1)
    # heads (strides 8, 16, 32) with bottom-up path
    v4_extra = (("iou_thresh", "0.213"), ("cls_normalizer", "1.0"), ("iou_normalizer", "0.07"), ("iou_loss", "ciou"),
                ("nms_kind", "greedynms"), ("beta_nms", "0.6"))
    c.conv(256, 3)
    c.conv(nout, 1, act="linear", bn=0)
    c.yolo((0, 1, 2), COCO_ANCHORS_V4, classes, 9, (("scale_x_y", "1.2"),) + v4_extra)
    for mid, mask, back, sxy in ((256, (3, 4, 5), -16, "1.1"), (512, (6, 7, 8), -37, "1.05")):
        c.route(-4)
        c.conv(mid, 3, 2)
        c.route(-1, back)
        for _ in range(3):
            c.conv(mid, 1)
            c.conv(mid * 2, 3)
        c.conv(nout, 1, act="linear", bn=0)
        c.yolo(mask, COCO_ANCHORS_V4, classes, 9, (("scale_x_y", sxy),) + v4_extra)
    return c.text()


def yolov3_mobilenet(classes=80):
    """YOLOv3 head on a MobileNetV3-large backbone (the reference's cfg/yolov3-mobilenet/yolov3-mobilenet-coco.cfg):
    inverted-residual blocks = 1x1 expand -> depthwise k x k -> [squeeze-excite] -> 1x1 project (linear) [+ shortcut]."""
    c = _Cfg([("batch", 16), ("subdivisions", 1)] + _net()[2:])
    nout = 3 * (classes + 5)
    c.conv(16, 3, 2, act="h_swish")
    # (expansion, out, kernel, stride, se, activation, residual)
    blocks = ((16, 16, 3, 1, 0, "relu6", 1), (64, 24, 3, 2, 0, "relu6", 0), (72, 24, 3, 1, 0, "relu6", 1),
              (72, 40, 5, 2, 1, "relu6", 0), (120, 40, 5, 1, 1, "relu6", 1), (120, 40, 5, 1, 1, "relu6", 1),
              (240, 80, 3, 2, 0, "h_swish", 0), (200, 80, 3, 1, 0, "h_swish", 1), (184, 80, 3, 1, 0, "h_swish", 1),
              (184, 80, 3, 1, 0, "h_swish", 1), (480, 112, 3, 1, 1, "h_swish", 0), (672, 112, 3, 1, 1, "h_swish", 1),
              (672, 160, 5, 2, 1, "h_swish", 0), (960, 160, 5, 1, 1, "h_swish", 1), (960, 160, 5, 1, 1, "h_swish", 1))
    for exp, out, k, stride, se, act, res in blocks:
        c.conv(exp, 1, act=act)
        c.depthwise(exp, k, stride, act=act)
        if se:
            c.se(exp)
        c.conv(out, 1, act="linear")
        if res:
            c.shortcut(-5 if se else -4)
    c.conv(1024, 1, act="h_swish")
    for scale, (mid, mask, skip) in enumerate(((512, (6, 7, 8), None), (256, (3, 4, 5), 49), (128, (0, 1, 2), 25))):
        if skip is not None:
            c.route(-4)
            c.conv(mid, 1)
            c.upsample(2)
            c.route(-1, skip)
        for _ in range(3):
            c.conv(mid, 1)
            c.conv(mid * 2, 3)
        c.conv(nout, 1, act="linear", bn=0)
        c.yolo(mask, COCO_ANCHORS_V3, classes, 9, (("random", 1),))
    return c.text()


def yolov3_ghost(classes=80):
    """YOLOv3 head on a GhostNet backbone (the reference's cfg/yolov3-ghostnet/yolov3-ghost-coco.cfg).  A ghost module is
    a 1x1 primary conv, a 3x3 depthwise cheap operation ([convolutional] groups=C) and a concat of the two; a bottleneck
    is an expanding ghost module, a k x k stride-2 depthwise conv when it downsamples, [se], and a linear ghost module,
    with a shortcut from its input, through a depthwise conv and a 1x1 conv where the width or the size changes."""
    c = _Cfg([("batch", 16), ("subdivisions", 1)] + _net()[2:])
    nout = 3 * (classes + 5)

    def conv(filters, size, stride=1, act="none", groups=1):
        return c.block("convolutional", ("batch_normalize", 1), ("filters", filters), ("size", size), ("stride", stride),
                       ("pad", size // 2), ("groups", groups), ("activation", act))

    def ghost(half, act):
        primary = conv(half, 1, act=act)
        conv(half, 3, act=act, groups=half)
        return c.route(-1, primary)

    width = 16
    start = conv(width, 3, 2, act="relu")
    # (expanded half width, output half width, kernel, stride, se, shortcut block without its activation key)
    blocks = ((8, 8, 3, 1, 0, 0), (24, 12, 3, 2, 0, 0), (36, 12, 3, 1, 0, 0), (36, 20, 5, 2, 1, 0), (60, 20, 3, 1, 1, 1),
              (120, 40, 3, 2, 0, 0), (100, 40, 3, 1, 0, 0), (92, 40, 3, 1, 0, 0), (92, 40, 3, 1, 0, 0),
              (240, 56, 3, 1, 1, 0), (336, 56, 3, 1, 1, 0), (336, 80, 5, 2, 1, 0), (480, 80, 3, 1, 0, 0),
              (480, 80, 3, 1, 1, 0), (480, 80, 3, 1, 0, 0), (480, 80, 3, 1, 1, 1))
    for exp, out, k, stride, se, bare in blocks:
        ghost(exp, "relu")
        if stride == 2:
            conv(2 * exp, k, 2, groups=2 * exp)
        if se:
            c.block("se", ("reduction", 4))
        end = ghost(out, "none")
        frm = start
        if stride == 2 or 2 * out != width:     # the projected input is added to the block's output
            c.route(start)
            conv(width, k, stride, groups=width)
            conv(2 * out, 1)
            frm = end
        c.block("shortcut", ("from", frm - c.n), *(() if bare else (("activation", "none"),)))
        start, width = c.n - 1, 2 * out
    conv(960, 1, act="relu")
    for scale, (mid, mask, skip) in enumerate(((512, (6, 7, 8), None), (256, (3, 4, 5), 96), (128, (0, 1, 2), 45))):
        if skip is not None:
            c.route(-4)
            conv(mid, 1, act="leaky")
            c.upsample(2)
            c.route(-1, skip)
        for _ in range(3):
            conv(mid, 1, act="leaky")
            conv(mid * 2, 3, act="leaky")
        c.block("convolutional", ("size", 1), ("stride", 1), ("pad", 0), ("filters", nout), ("groups", 1),
                ("activation", "linear"))
        c.yolo(mask, COCO_ANCHORS_V3, classes, 9, (("random", 1),))
    return c.text()


def _v2_head(c, classes):
    """One stride-32 head over all five anchors: 5 * (classes + 5) filters (425 for 80 classes)."""
    c.conv(5 * (classes + 5), 1, act="linear", bn=0)
    c.yolo((0, 1, 2, 3, 4), V2_ANCHORS, classes, 5, (("random", 1),))


def yolov2(classes=80):
    """Darknet-19 (3x3 convs doubling the width per stage, 1x1 bottlenecks at half width between them, 2x2 max-pools)
    with three 3x3 x 1024 convs before the head."""
    c = _Cfg(_net(608, 608))
    for stage, (filters, pairs) in enumerate(((32, 0), (64, 0), (128, 1), (256, 1), (512, 2), (1024, 2))):
        c.conv(filters, 3)
        for _ in range(pairs):
            c.conv(filters // 2, 1)
            c.conv(filters, 3)
        if stage < 5:
            c.maxpool(2, 2)
    for _ in range(3):
        c.conv(1024, 3)
    _v2_head(c, classes)
    return c.text()


def yolov2_tiny(classes=80):
    """Six 3x3 conv + 2x2 max-pool pairs (the last pool with stride 1), two 3x3 x 1024 convs, the head."""
    c = _Cfg(_net())
    for i, f in enumerate((16, 32, 64, 128, 256, 512)):
        c.conv(f, 3)
        c.maxpool(2, 2 if i < 5 else 1)
    c.conv(1024, 3)
    c.conv(1024, 3)
    _v2_head(c, classes)
    return c.text()


ARCHS = {"yolov3": yolov3, "yolov3-tiny": yolov3_tiny, "yolov4": yolov4, "yolov3-mobilenet": yolov3_mobilenet,
         "yolov3-ghost": yolov3_ghost, "yolov2": yolov2, "yolov2-tiny": yolov2_tiny}


def cfg_text(name, classes=80):
    return ARCHS[name](classes)


def write_cfg(name, directory, classes=80):
    """Write <directory>/<name>.cfg (file name keeps 'yolov4' in the path: models.py keys the stride order on it)."""
    import os
    os.makedirs(directory, exist_ok=True)
    path = os.path.join(directory, name + ".cfg")
    # write-then-rename: several ranks may generate the same file concurrently; a reader never sees a truncated cfg
    tmp = "%s.%d.tmp" % (path, os.getpid())
    with open(tmp, "w") as f:
        f.write(cfg_text(name, classes))
    os.replace(tmp, path)
    return path
