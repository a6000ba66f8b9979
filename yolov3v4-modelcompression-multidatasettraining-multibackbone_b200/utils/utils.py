"""Loss slice of the reference's utils/utils.py under the same names, executed by the sm_90a kernels:

    compute_loss(p, targets, model)   reference utils/utils.py:368-432
    build_targets(p, targets, model)  reference utils/utils.py:725-779
    bbox_iou / wh_iou                 reference utils/utils.py:254-297, 325-330
    FocalLoss / smooth_BCE            reference utils/utils.py:333-365
    non_max_suppression(...)          reference utils/utils.py:782-860   (csrc/nms.cu, whole batch on the device)
    xywh2xyxy / xyxy2xywh / box_iou / clip_coords   reference utils/utils.py:118-159, 300-322 (tensor helpers)
    compute_lost_KD / KD2 / KD3       reference utils/utils.py:435-520   (csrc/kd.cu)

Everything else of the reference's utils/utils.py (AP, plotting, KD losses, dataset helpers) is outside the
accelerated hot path; with B2Y_REFERENCE_ROOT set those names are re-exported from the reference's own file so
train.py / test.py keep working unchanged (INTEGRATION.md).
"""
import glob  # noqa: F401  (star-import surface of the reference module)
import importlib.util as _ilu
import math
import os
import random  # noqa: F401
import shutil  # noqa: F401
import subprocess  # noqa: F401
import time  # noqa: F401
from copy import copy  # noqa: F401
from pathlib import Path  # noqa: F401
from sys import platform  # noqa: F401

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F  # noqa: F401

from . import torch_utils  # noqa: F401

# ---- overlay: non-hot-path names come from the reference's own utils/utils.py when it is available -----------
_ref_root = os.environ.get("B2Y_REFERENCE_ROOT", "")
_ref_file = os.path.join(_ref_root, "utils", "utils.py") if _ref_root else ""
if _ref_file and os.path.isfile(_ref_file):
    _spec = _ilu.spec_from_file_location("utils._reference_utils", _ref_file)
    _mod = _ilu.module_from_spec(_spec)
    _mod.__package__ = "utils"
    _spec.loader.exec_module(_mod)
    globals().update({k: v for k, v in vars(_mod).items() if not k.startswith("__")})

_PARALLEL = (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel)


def smooth_BCE(eps=0.1):
    """positive / negative BCE targets under label smoothing."""
    return 1.0 - 0.5 * eps, 0.5 * eps


class FocalLoss(nn.Module):
    """Focal modulation of a BCEWithLogits criterion, active when hyp['fl_gamma'] > 0.  compute_loss runs it inside the
    fused loss kernel (csrc/yolo.cu focal_modulate); this module is the tensor form for callers outside it."""

    def __init__(self, loss_fcn, gamma=1.5, alpha=0.25):
        super().__init__()
        self.loss_fcn, self.gamma, self.alpha = loss_fcn, gamma, alpha
        self.reduction = loss_fcn.reduction
        self.loss_fcn.reduction = 'none'

    def forward(self, pred, true):
        loss = self.loss_fcn(pred, true)
        prob = torch.sigmoid(pred)
        p_t = true * prob + (1 - true) * (1 - prob)
        loss = loss * (true * self.alpha + (1 - true) * (1 - self.alpha)) * (1.0 - p_t) ** self.gamma
        if self.reduction == 'mean':
            return loss.mean()
        return loss.sum() if self.reduction == 'sum' else loss


def wh_iou(wh1, wh2):
    """[N,2] x [M,2] -> [N,M] IoU of boxes sharing a corner."""
    a, b = wh1[:, None], wh2[None]
    inter = torch.min(a, b).prod(2)
    return inter / (a.prod(2) + b.prod(2) - inter)


def bbox_iou(box1, box2, x1y1x2y2=True, GIoU=False, DIoU=False, CIoU=False):
    """IoU family of box1 (4,n) against box2 (n,4); tensor helper for callers outside the fused loss
    (the fused kernel csrc/yolo.cu:giou_fwd_bwd implements the GIoU branch with identical eps placement)."""
    box2 = box2.t()
    if x1y1x2y2:
        ax1, ay1, ax2, ay2 = box1[0], box1[1], box1[2], box1[3]
        bx1, by1, bx2, by2 = box2[0], box2[1], box2[2], box2[3]
    else:
        ax1, ax2 = box1[0] - box1[2] / 2, box1[0] + box1[2] / 2
        ay1, ay2 = box1[1] - box1[3] / 2, box1[1] + box1[3] / 2
        bx1, bx2 = box2[0] - box2[2] / 2, box2[0] + box2[2] / 2
        by1, by2 = box2[1] - box2[3] / 2, box2[1] + box2[3] / 2
    inter = (torch.min(ax2, bx2) - torch.max(ax1, bx1)).clamp(0) * (torch.min(ay2, by2) - torch.max(ay1, by1)).clamp(0)
    w1, h1, w2, h2 = ax2 - ax1, ay2 - ay1, bx2 - bx1, by2 - by1
    union = (w1 * h1 + 1e-16) + w2 * h2 - inter
    iou = inter / union
    if not (GIoU or DIoU or CIoU):
        return iou
    cw = torch.max(ax2, bx2) - torch.min(ax1, bx1)
    ch = torch.max(ay2, by2) - torch.min(ay1, by1)
    if GIoU:
        c_area = cw * ch + 1e-16
        return iou - (c_area - union) / c_area
    c2 = cw ** 2 + ch ** 2 + 1e-16
    rho2 = ((bx1 + bx2) - (ax1 + ax2)) ** 2 / 4 + ((by1 + by2) - (ay1 + ay2)) ** 2 / 4
    if DIoU:
        return iou - rho2 / c2
    v = (4 / math.pi ** 2) * torch.pow(torch.atan(w2 / h2) - torch.atan(w1 / h1), 2)
    with torch.no_grad():
        alpha = v / (1 - iou + v)
    return iou - (rho2 / c2 + v * alpha)


def _unwrap(model):
    return model.module if type(model) in _PARALLEL else model


def _yolo_modules(model):
    base = _unwrap(model)
    return [base.module_list[j] for j in model.yolo_layers]


def _device_anchor_vec(layer, device):
    av = layer.anchor_vec
    if av.device != device:
        layer.anchor_vec = av = av.to(device)
        layer.anchor_wh = layer.anchor_wh.to(device)
    return av.float().contiguous()


def build_targets(p, targets, model):
    """Anchor matching per yolo layer -> (tcls, tbox, indices=(b, a, gj, gi), anchor_vec[a]); same ordering as the
    reference (anchor-major, target-minor, filtered by wh_iou > hyp['iou_t']), computed by b2y_build_targets."""
    from b200yolo import ops
    if not targets.is_cuda:
        raise RuntimeError("build_targets runs on the CUDA device only (no CPU fallback)")
    tcls, tbox, indices, av = [], [], [], []
    for i, layer in enumerate(_yolo_modules(model)):
        anchors = _device_anchor_vec(layer, targets.device)
        B, ny, nx = int(p[i].shape[0]), int(p[i].shape[2]), int(p[i].shape[3])
        idx, box, cls = ops.build_targets_layer(targets, anchors, B, ny, nx, model.hyp['iou_t'])
        if cls.numel():
            assert int(cls.max()) < model.nc, \
                'Model accepts %g classes labeled from 0-%g, however you labelled a class %g. ' \
                'See https://github.com/ultralytics/yolov3/wiki/Train-Custom-Data' % (model.nc, model.nc - 1, cls.max())
        indices.append((idx[0], idx[1], idx[2], idx[3]))
        tbox.append(box)
        tcls.append(cls)
        av.append(anchors[idx[1]])
    return tcls, tbox, indices, av


class _YoloLoss(torch.autograd.Function):
    """loss and d(loss)/d(p_i) for all yolo layers in one shot (kernels: csrc/yolo.cu loss_*_kernel)."""

    @staticmethod
    def forward(ctx, targets, cfg, *preds):
        from b200yolo import ops
        anchors, hyp, gr, nc = cfg
        need_grad = any(t.requires_grad for t in preds)
        dev = preds[0].device
        lbox = torch.zeros(1, device=dev)
        lobj = torch.zeros(1, device=dev)
        lcls = torch.zeros(1, device=dev)
        grads = []
        for pi, av in zip(preds, anchors):
            cells = pi.numel() // pi.shape[-1]
            out4, dp = ops.yolo_loss_layer(pi.float(), targets, av, hyp['iou_t'], gr, hyp['cls_pw'], hyp['obj_pw'],
                                           hyp['giou'], hyp['obj'], hyp['cls'] if nc > 1 else 0.0,
                                           want_grad=need_grad, fl_gamma=hyp.get('fl_gamma', 0))
            nb = out4[1]
            has = (nb > 0).float()
            denom = nb.clamp(min=1.0)
            lbox += has * out4[0] / denom
            if nc > 1:
                lcls += has * out4[2] / (denom * nc)
            lobj += out4[3] / cells
            grads.append(dp)
        lbox *= hyp['giou']
        lobj *= hyp['obj']
        lcls *= hyp['cls']
        ctx.grads = grads
        ctx.dtypes = [t.dtype for t in preds]
        loss = lbox + lobj + lcls
        items = torch.cat((lbox, lobj, lcls, loss)).detach()
        ctx.mark_non_differentiable(items)
        return loss, items

    @staticmethod
    def backward(ctx, g_loss, _g_items):
        outs = []
        for dp, dt in zip(ctx.grads, ctx.dtypes):
            outs.append(None if dp is None else (dp * g_loss).to(dt))
        return (None, None) + tuple(outs)


def compute_loss(p, targets, model):
    """GIoU box + objectness + class loss of the YOLO head; returns (loss[1], cat(lbox, lobj, lcls, loss).detach()).
    hyp['fl_gamma'] > 0 wraps the class and objectness BCE in the focal loss, as the reference does."""
    if not p[0].is_cuda:
        raise RuntimeError("compute_loss runs on the CUDA device only (no CPU fallback)")
    h = model.hyp
    dev = p[0].device
    anchors = [_device_anchor_vec(m, dev) for m in _yolo_modules(model)]
    t = targets.to(dev).float()
    _check_class_ids(t, int(model.nc))
    return _YoloLoss.apply(t, (anchors, h, float(model.gr), int(model.nc)), *p)


# The reference asserts "class id < nc" inside build_targets (utils/utils.py:775) with a blocking .max() on the
# device tensor.  A blocking read here would stall the launch queue once per training step (the CPU could no longer
# run ahead of the GPU), so the maximum is copied to pinned host memory asynchronously and verified when it has
# arrived -- at the latest at the start of the NEXT compute_loss call -- with the reference's message.
_pending_check = None


def _raise_bad_class(nc, cmax):
    raise AssertionError('Model accepts %g classes labeled from 0-%g, however you labelled a class %g. '
                         'See https://github.com/ultralytics/yolov3/wiki/Train-Custom-Data' % (nc, nc - 1, cmax))


def _check_class_ids(t, nc):
    global _pending_check
    if _pending_check is not None:
        host, ev, pnc = _pending_check
        ev.synchronize()
        _pending_check = None
        if float(host[0]) >= pnc:
            _raise_bad_class(pnc, float(host[0]))
    if not t.numel():
        return
    if torch.cuda.is_current_stream_capturing():
        return
    host = torch.empty(1, dtype=torch.float32).pin_memory()
    host.copy_(t[:, 1].max().reshape(1), non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    if ev.query():                      # already there (small queue): behave exactly like the reference
        if float(host[0]) >= nc:
            _raise_bad_class(nc, float(host[0]))
        return
    _pending_check = (host, ev, nc)


def flush_checks():
    """Force the deferred class-id check of the last compute_loss call (raises like the reference if it failed)."""
    _check_class_ids(torch.zeros(0, 6), 0)


# ---- detection post-processing (SURVEY section 8 f1) -------------------------------------------------------------------
def xyxy2xywh(x):
    """[n, 4] corner boxes -> (centre x, centre y, width, height)."""
    y = torch.zeros_like(x) if isinstance(x, torch.Tensor) else np.zeros_like(x)
    y[:, 0] = (x[:, 0] + x[:, 2]) / 2
    y[:, 1] = (x[:, 1] + x[:, 3]) / 2
    y[:, 2] = x[:, 2] - x[:, 0]
    y[:, 3] = x[:, 3] - x[:, 1]
    return y


def xywh2xyxy(x):
    """[n, 4] (centre x, centre y, width, height) -> corner boxes."""
    y = torch.zeros_like(x) if isinstance(x, torch.Tensor) else np.zeros_like(x)
    y[:, 0] = x[:, 0] - x[:, 2] / 2
    y[:, 1] = x[:, 1] - x[:, 3] / 2
    y[:, 2] = x[:, 0] + x[:, 2] / 2
    y[:, 3] = x[:, 1] + x[:, 3] / 2
    return y


def clip_coords(boxes, img_shape):
    """Clamp corner boxes in place to an image of shape (height, width)."""
    for col, hi in ((0, img_shape[1]), (1, img_shape[0]), (2, img_shape[1]), (3, img_shape[0])):
        boxes[:, col].clamp_(0, hi)


def box_iou(box1, box2):
    """[N, 4] x [M, 4] corner boxes -> [N, M] IoU."""
    a1 = (box1[:, 2] - box1[:, 0]) * (box1[:, 3] - box1[:, 1])
    a2 = (box2[:, 2] - box2[:, 0]) * (box2[:, 3] - box2[:, 1])
    inter = (torch.min(box1[:, None, 2:], box2[:, 2:]) - torch.max(box1[:, None, :2], box2[:, :2])).clamp(0).prod(2)
    return inter / (a1[:, None] + a2 - inter)


def non_max_suppression(prediction, conf_thres=0.1, iou_thres=0.6, multi_label=True, classes=None, agnostic=False):
    """Batched NMS on the device with the reference's candidate order, tie-breaking and merge refinement
    (b200yolo/detect.py -> csrc/nms.cu).  Returns a list of [n, 6] (x1, y1, x2, y2, conf, cls) tensors or None."""
    from b200yolo import detect
    return detect.non_max_suppression(prediction, conf_thres, iou_thres, multi_label, classes, agnostic)


# ---- knowledge distillation (SURVEY section 8 f4) ------------------------------------------------------------------------
def compute_lost_KD(output_s, output_t, num_classes, batch_size):
    from b200yolo import kd
    return kd.compute_lost_KD(output_s, output_t, num_classes, batch_size)


def compute_lost_KD2(model, targets, output_s, output_t):
    from b200yolo import kd
    return kd.compute_lost_KD2(model, targets, output_s, output_t)


def compute_lost_KD3(model, targets, output_s, output_t):
    from b200yolo import kd
    return kd.compute_lost_KD3(model, targets, output_s, output_t)
