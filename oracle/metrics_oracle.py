"""TEST INFRASTRUCTURE ONLY (never imported by the product path).

CPU restatement of the reference's detection post-processing and mAP bookkeeping, used to check that the H100 engine's
predictions give the same mAP as the reference's on a held synthetic batch (BASELINE north_star: |dmAP| <= 1e-4):

  * nms()            <- utils/utils.py:782-860  non_max_suppression (multi-label candidates, per-class offset boxes,
                        torchvision NMS, 'merge' box refinement for 1 < n < 3000)
  * match_image()    <- test.py:123-170         per-image TP matrix over the 10 IoU thresholds 0.5:0.05:0.95
  * ap_per_class()   <- utils/utils.py:162-219  precision / recall curves per class, P/R read at conf 0.1
  * average_precision() <- utils/utils.py:222-251  envelope + 101-point interpolation

Pinned against outputs of the reference itself: tests/golden/map_case.npz (oracle/gen_golden_map.py),
tests/test_oracle_golden.py::test_metrics_oracle_matches_reference.
"""
import numpy as np
import torch
import torchvision

MIN_WH, MAX_WH = 2, 4096          # utils.py:790
IOU_THRESHOLDS = torch.linspace(0.5, 0.95, 10)   # test.py:66


def xywh_to_xyxy(b):
    """utils.py:138-146"""
    out = torch.zeros_like(b)
    half = b[:, 2:4] / 2
    out[:, 0:2] = b[:, 0:2] - half
    out[:, 2:4] = b[:, 0:2] + half
    return out


def pairwise_iou(a, b):
    """utils.py:300-322: IoU of every box of a (N,4 xyxy) with every box of b (M,4)."""
    area_a = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt = torch.max(a[:, None, :2], b[None, :, :2])
    rb = torch.min(a[:, None, 2:], b[None, :, 2:])
    inter = (rb - lt).clamp(0).prod(2)
    return inter / (area_a[:, None] + area_b[None, :] - inter)


def nms(prediction, conf_thres=0.1, iou_thres=0.6, multi_label=True, classes=None, agnostic=False):
    """prediction [B, rows, 5+nc] (xywh px, obj, cls probs) -> list of [n, 6] (xyxy, conf, cls) or None per image."""
    nc = prediction.shape[2] - 5
    multi = multi_label and nc > 1
    results = [None] * prediction.shape[0]
    for bi in range(prediction.shape[0]):
        x = prediction[bi]
        x = x[x[:, 4] > conf_thres]
        wh = x[:, 2:4]
        x = x[((wh > MIN_WH) & (wh < MAX_WH)).all(1)]
        if x.shape[0] == 0:
            continue
        x = x.clone()
        x[:, 5:] = x[:, 5:] * x[:, 4:5]                 # conf = obj * cls (utils.py:809)
        box = xywh_to_xyxy(x[:, :4])
        if multi:
            rows, cls = (x[:, 5:] > conf_thres).nonzero(as_tuple=False).t()
            det = torch.cat((box[rows], x[rows, cls + 5].unsqueeze(1), cls.float().unsqueeze(1)), 1)
        else:
            conf, cls = x[:, 5:].max(1)
            det = torch.cat((box, conf.unsqueeze(1), cls.float().unsqueeze(1)), 1)
        if classes:                                        # utils.py:823-824
            det = det[(det[:, 5:6] == torch.tensor(classes, dtype=det.dtype)).any(1)]
        det = det[torch.isfinite(det).all(1)]
        n = det.shape[0]
        if n == 0:
            continue
        offs = det[:, 5:6] * 0 if agnostic else det[:, 5:6]
        shifted = det[:, :4] + offs * MAX_WH              # per-class offset so one NMS call handles all classes
        scores = det[:, 4]
        keep = torchvision.ops.nms(shifted, scores, iou_thres)
        if 1 < n < 3000:                                  # 'merge': score-weighted mean of the overlapping boxes
            w = (pairwise_iou(shifted[keep], shifted) > iou_thres) * scores[None]
            det[keep, :4] = torch.mm(w, det[:, :4]).float() / w.sum(1, keepdim=True)
        results[bi] = det[keep]
    return results


def match_image(pred, labels):
    """pred [n,6] (xyxy, conf, cls); labels [m,5] (cls, xyxy).  -> bool [n,10]: true positive at each IoU threshold.
    A target can be claimed once; predictions are visited in their given order within each class (test.py:150-170)."""
    correct = torch.zeros(pred.shape[0], IOU_THRESHOLDS.numel(), dtype=torch.bool)
    if labels.shape[0] == 0:
        return correct
    tcls = labels[:, 0]
    claimed = []
    for c in torch.unique(tcls):
        ti = (tcls == c).nonzero(as_tuple=False).view(-1)
        pi = (pred[:, 5] == c).nonzero(as_tuple=False).view(-1)
        if pi.numel() == 0:
            continue
        best, arg = pairwise_iou(pred[pi, :4], labels[ti, 1:5]).max(1)
        for j in (best > IOU_THRESHOLDS[0]).nonzero(as_tuple=False):
            d = ti[arg[j]]
            if d not in claimed:
                claimed.append(d)
                correct[pi[j]] = best[j] > IOU_THRESHOLDS
                if len(claimed) == labels.shape[0]:
                    break
    return correct


def average_precision(recall, precision):
    mrec = np.concatenate(([0.0], recall, [min(recall[-1] + 1e-3, 1.0)]))
    mpre = np.concatenate(([0.0], precision, [0.0]))
    mpre = np.flip(np.maximum.accumulate(np.flip(mpre)))
    grid = np.linspace(0, 1, 101)
    trapezoid = getattr(np, "trapezoid", None) or np.trapz          # numpy >= 2 renamed trapz
    return trapezoid(np.interp(grid, mrec, mpre), grid)


def ap_per_class(tp, conf, pred_cls, target_cls, pr_score=0.1):
    order = np.argsort(-conf)
    tp, conf, pred_cls = tp[order], conf[order], pred_cls[order]
    classes = np.unique(target_cls)
    shape = (len(classes), tp.shape[1])
    ap, p, r = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    for k, c in enumerate(classes):
        sel = pred_cls == c
        n_gt, n_p = (target_cls == c).sum(), sel.sum()
        if n_gt == 0 or n_p == 0:
            continue
        fp_cum = (1 - tp[sel]).cumsum(0)
        tp_cum = tp[sel].cumsum(0)
        recall = tp_cum / (n_gt + 1e-16)
        precision = tp_cum / (tp_cum + fp_cum)
        r[k] = np.interp(-pr_score, -conf[sel], recall[:, 0])
        p[k] = np.interp(-pr_score, -conf[sel], precision[:, 0])
        for j in range(tp.shape[1]):
            ap[k, j] = average_precision(recall[:, j], precision[:, j])
    return p, r, ap, classes.astype("int32")


def clip_boxes(det, height, width):
    """utils.py:149-159 clip_coords: xyxy boxes clamped to the image (test.py:137)."""
    det[:, 0].clamp_(0, width)
    det[:, 1].clamp_(0, height)
    det[:, 2].clamp_(0, width)
    det[:, 3].clamp_(0, height)


def mean_ap(prediction, labels_per_image, conf_thres, iou_thres, height, width):
    """Full pipeline of test.py:118-190: NMS -> clip -> matching -> AP.  labels_per_image: list of [m,5]
    (cls, xyxy px) tensors (or None).  Returns (mAP@0.5, mAP@0.5:0.95, number of detections)."""
    dets = nms(prediction.float().cpu(), conf_thres, iou_thres)
    stats = []
    for det, lab in zip(dets, labels_per_image):
        if det is not None:
            clip_boxes(det, height, width)
        nl = 0 if lab is None else lab.shape[0]
        tcls = lab[:, 0].tolist() if nl else []
        if det is None:
            if nl:
                stats.append((torch.zeros(0, 10, dtype=torch.bool), torch.Tensor(), torch.Tensor(), tcls))
            continue
        correct = match_image(det, lab) if nl else torch.zeros(det.shape[0], 10, dtype=torch.bool)
        stats.append((correct, det[:, 4], det[:, 5], tcls))
    cols = [np.concatenate([np.asarray(t) for t in col], 0) for col in zip(*stats)]
    p, r, ap, _ = ap_per_class(*cols)
    return float(ap[:, 0].mean()), float(ap.mean(1).mean()), int(cols[0].shape[0])
