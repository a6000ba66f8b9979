"""Knowledge-distillation losses of the YOLO head on the device (SURVEY section 8 f4), csrc/kd.cu.

    compute_lost_KD(output_s, output_t, num_classes, batch_size)      utils/utils.py:435-444   (train.py --KDstr 1)
    compute_lost_KD2(model, targets, output_s, output_t)              utils/utils.py:447-490   (--KDstr 2)
    compute_lost_KD3(model, targets, output_s, output_t)              utils/utils.py:493-520   (--KDstr 3)

The reference composes each of them from ~15 ATen ops per yolo layer over the full prediction tensors (log_softmax,
softmax, KLDivLoss, gathers) and lets autograd replay them backwards.  Here the value and the gradient w.r.t. the
student's predictions come from one pass per layer (plus one tiny kernel for the matched cells); the teacher is a
constant (train.py runs it in eval mode and never steps its parameters).  KD strategies 4 - 6 (feature imitation on
the intermediate feature maps) are not part of this path.
"""
import ctypes as C

import torch

from .lib import call, ptr, stream_ptr

T_KD = 3.0      # utils.py:436, 449, 494


def _soft(ps, pt, col0, grad_scale, acc, want_grad):
    """acc[0] += KL sum over all cells of one layer; returns the gradient buffer (zeros outside the softmax columns)."""
    s = ps.detach().float().contiguous()
    t = pt.detach().float().contiguous()
    no = s.shape[-1]
    ds = torch.zeros_like(s) if want_grad else None
    call("b2y_kd_soft_rows", ptr(s), ptr(t), C.c_longlong(s.numel() // no), no, col0, no - col0, T_KD, float(grad_scale),
         ptr(acc), ptr(ds), stream_ptr())
    return s, t, ds


class _KD(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mode, cfg, targets, n, *tensors):
        from . import ops
        out_s, out_t = tensors[:n], tensors[n:]
        dev = out_s[0].device
        want = any(t.requires_grad for t in out_s)
        acc = torch.zeros(2, dtype=torch.float64, device=dev)        # [soft-target sum (scaled), box sum]
        reg = torch.zeros(2, dtype=torch.int32, device=dev)
        grads, reg_nb = [], 0
        if mode == 1:
            num_classes, batch_size = cfg
            k = T_KD * T_KD / float(batch_size) * 0.001              # * (T * T) / batch_size * Lambda_ST
            cls_acc = torch.zeros(1, dtype=torch.float64, device=dev)
            for ps, pt in zip(out_s, out_t):
                assert ps.shape[-1] == num_classes + 5
                grads.append(_soft(ps, pt, 0, k, cls_acc, want)[2])
            loss = (cls_acc * k).float().reshape(())
        else:
            anchors, iou_t, nc = cfg
            l_cls, l_box = (1e-4, 1e-3)                              # Lambda_cls, Lambda_box (utils.py:450, 495)
            layer_acc = torch.zeros(len(out_s), dtype=torch.float64, device=dev)
            scales = []
            for i, (ps, pt, av) in enumerate(zip(out_s, out_t, anchors)):
                k = T_KD * T_KD / float(ps.shape[0]) * l_cls         # * (T * T) / ps.size(0), then * Lambda_cls
                scales.append(k)
                s, t, ds = _soft(ps, pt, 4, k, layer_acc[i:i + 1], want)
                B, na, ny, nx, no = s.shape
                idx, tbox, _ = ops.build_targets_layer(targets, av, B, ny, nx, iou_t)
                nb = int(idx.shape[1])
                reg_nb += nb
                if nb:
                    call("b2y_kd_box", ptr(s), ptr(t), ptr(idx.contiguous()), ptr(tbox.contiguous()), ptr(av), nb, na,
                         ny, nx, no, 2 if mode == 2 else 3, 0.0, l_box, ptr(acc[1:2]), ptr(reg[0:1]), ptr(ds),
                         stream_ptr())
                grads.append(ds)
            lcls = (layer_acc * torch.tensor(scales, dtype=torch.float64, device=dev)).sum()
            loss = (lcls + acc[1] * l_box).float().reshape(1)
        ctx.grads = grads
        ctx.dtypes = [t.dtype for t in out_s]
        ctx.n = n
        counts = torch.stack((reg[0].double(), torch.tensor(float(reg_nb), dtype=torch.float64, device=dev)))
        ctx.mark_non_differentiable(counts)
        return loss, counts          # (reg_num, reg_nb): the caller forms the ratio in Python like the reference

    @staticmethod
    def backward(ctx, g, _g_counts):
        outs = [None if d is None else (d * g).to(dt) for d, dt in zip(ctx.grads, ctx.dtypes)]
        return (None, None, None, None) + tuple(outs) + (None,) * ctx.n


def _check(output_s, output_t):
    if not output_s[0].is_cuda:
        raise RuntimeError("the KD losses run on the CUDA device only (no CPU fallback)")
    assert len(output_s) == len(output_t) and all(a.shape == b.shape for a, b in zip(output_s, output_t))


def compute_lost_KD(output_s, output_t, num_classes, batch_size):
    """Soft-target loss over the whole 5 + nc prediction row of every cell (utils.py:435-444)."""
    _check(output_s, output_t)
    return _KD.apply(1, (int(num_classes), int(batch_size)), None, len(output_s), *output_s, *output_t)[0]


def _kd_matched(mode, model, targets, output_s, output_t):
    from utils import utils as U
    _check(output_s, output_t)
    dev = output_s[0].device
    anchors = [U._device_anchor_vec(m, dev) for m in U._yolo_modules(model)]
    t = targets.to(dev).float()
    U._check_class_ids(t, int(model.nc))
    cfg = (anchors, float(model.hyp['iou_t']), int(model.nc))
    return _KD.apply(mode, cfg, t, len(output_s), *output_s, *output_t)


def compute_lost_KD2(model, targets, output_s, output_t):
    """Soft targets on (objectness, classes) + box regression towards the labels where the student is further from them
    than the teacher (utils.py:447-490).  Returns (loss[1], reg_ratio)."""
    loss, counts = _kd_matched(2, model, targets, output_s, output_t)
    reg_num, reg_nb = counts.tolist()    # the reference syncs here as well (.item(), utils.py:476)
    return loss, (reg_num / reg_nb if reg_nb else 0)


def compute_lost_KD3(model, targets, output_s, output_t):
    """Soft targets on (objectness, classes) + squared distance to the teacher's boxes on the matched cells
    (utils.py:493-520)."""
    return _kd_matched(3, model, targets, output_s, output_t)[0]
