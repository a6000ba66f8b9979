"""ORACLE -- test infrastructure only.  The reference's compute_loss (utils/utils.py:368-432) with its focal-loss branch:
hyp['fl_gamma'] > 0 wraps BOTH criteria, BCEcls and BCEobj, in FocalLoss(., gamma) with alpha 0.25
(utils/utils.py:333-360, 383-385).  Box targets, GIoU and build_targets are darknet_oracle's.

Pinned: tests/test_host_heads.py checks it against tests/golden/focal_case.npz, which oracle/gen_golden_heads.py
produced by running the reference itself.
"""
import torch

from . import darknet_oracle as orc


def focal(bce_none, gamma, alpha=0.25):
    """FocalLoss.forward (utils.py:342-360) with reduction 'mean': the element-wise BCE (reduction 'none') times the
    alpha factor and (1 - p_t) ** gamma, then the mean."""
    def crit(pred, true):
        loss = bce_none(pred, true)
        pred_prob = torch.sigmoid(pred)
        p_t = true * pred_prob + (1 - true) * (1 - pred_prob)
        alpha_factor = true * alpha + (1 - true) * (1 - alpha)
        modulating_factor = (1.0 - p_t) ** gamma
        loss = loss * (alpha_factor * modulating_factor)
        return loss.mean()
    return crit


def compute_loss(p, targets, anchor_vecs, hyp, nc, gr=1.0):
    """utils.py:368-432 with red='mean', smooth_BCE(eps=0) and hyp['fl_gamma'] > 0
    -> (loss[1], items[4] = lbox, lobj, lcls, loss).  With fl_gamma 0 it is darknet_oracle.compute_loss."""
    g = hyp.get('fl_gamma', 0.0)
    if not g > 0:
        return orc.compute_loss(p, targets, anchor_vecs, hyp, nc, gr)
    dev = p[0].device
    lcls, lbox, lobj = torch.zeros(1, device=dev), torch.zeros(1, device=dev), torch.zeros(1, device=dev)
    tcls, tbox, indices, av = orc.build_targets(p, targets, anchor_vecs, hyp['iou_t'])
    BCEcls = focal(torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor([hyp['cls_pw']], device=dev), reduction='none'), g)
    BCEobj = focal(torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor([hyp['obj_pw']], device=dev), reduction='none'), g)
    for i, pi in enumerate(p):
        b, a, gj, gi = indices[i]
        tobj = torch.zeros_like(pi[..., 0])
        nb = len(b)
        if nb:
            ps = pi[b, a, gj, gi]
            pxy = torch.sigmoid(ps[:, 0:2])
            pwh = torch.exp(ps[:, 2:4]).clamp(max=1E3) * av[i]
            giou = orc.giou_xywh(torch.cat((pxy, pwh), 1).t(), tbox[i])
            lbox = lbox + (1.0 - giou).mean()
            tobj[b, a, gj, gi] = (1.0 - gr) + gr * giou.detach().clamp(0).type(tobj.dtype)   # utils.py:407
            if nc > 1:
                t = torch.full_like(ps[:, 5:], 0.0)
                t[range(nb), tcls[i]] = 1.0
                lcls = lcls + BCEcls(ps[:, 5:], t)
        lobj = lobj + BCEobj(pi[..., 4], tobj)
    lbox = lbox * hyp['giou']
    lobj = lobj * hyp['obj']
    lcls = lcls * hyp['cls']
    loss = lbox + lobj + lcls
    return loss, torch.cat((lbox, lobj, lcls, loss)).detach()
