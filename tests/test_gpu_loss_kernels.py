"""The fused YOLO loss (b2y_yolo_loss) and target assignment (b2y_build_targets) against a float64 restatement of
compute_loss / build_targets (utils/utils.py:368-432, 725-779), at training-scale target counts and at the edges where
the kernels decide something: the wh_iou > iou_t threshold, cell boundaries, duplicate cells, saturated logits.

The match decision, the indices and tbox come from the reference's own fp32 arithmetic, run live on the CPU
(darknet_oracle.build_targets: wh_iou and targets * gain in float32); the kernel must reproduce them bit for bit.
The loss values and d loss / d p are then computed in float64 from those fp32 targets.

Gates: indices, classes and the match count nb exact; tbox bit-exact; loss items rel 1e-5; dp within
1e-5 * max|dp_ref| + 1e-7.  Candidates with an image index outside the batch or a cell off the grid, on which the
reference would raise an IndexError, are dropped by both kernels (and by the reference restatement here).
"""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import orc

HYP = dict(orc.DEFAULT_HYP)

# stock anchors in grid units (anchor_vec = anchors_px / stride)
V3 = [((10, 13), (16, 30), (33, 23)), ((30, 61), (62, 45), (59, 119)), ((116, 90), (156, 198), (373, 326))]
V4 = [((12, 16), (19, 36), (40, 28)), ((36, 75), (76, 55), (72, 146)), ((142, 110), (192, 243), (459, 401))]
V4_STRIDES = (8, 16, 32)
V2 = ((0.57273, 0.677385), (1.87446, 2.06253), (3.33843, 5.47434), (7.88282, 3.52778), (9.77052, 9.16828))


def _av(anchors_px, stride):
    return torch.tensor(anchors_px, dtype=torch.float32) / stride


def _f32(x):
    return np.float32(x)


# ---------------------------------------------------------------------------------------------------------------------
# edge-case constructors (host side, checked by test_boundary_constructor_matches_reference_expressions)
# ---------------------------------------------------------------------------------------------------------------------
def wh_iou_forms(aw, ah, gw, gh):
    """wh_iou of float32 anchor (aw, ah) vs float32 grid-unit target (gw, gh), emulated exactly in two roundings:
    'sep'   -- every product rounded on its own, as torch evaluates inter / (wh1.prod(2) + wh2.prod(2) - inter);
    'fused' -- gw * gh + (aw * ah) contracted into one FMA (one rounding of the exact sum), then - inter.
    Products of two float32 are exact in float64; the fused sum is checked to be exact in float64 before it is rounded
    to float32 once.  Returns (iou_sep, iou_fused, exact) as float32 arrays / a bool mask."""
    aw, ah, gw, gh = (np.asarray(v, dtype=np.float32) for v in (aw, ah, gw, gh))
    inter = np.minimum(aw, gw) * np.minimum(ah, gh)
    p1 = aw * ah
    sep = inter / ((p1 + gw * gh) - inter)
    prod = gw.astype(np.float64) * gh.astype(np.float64)
    s = prod + p1.astype(np.float64)
    bb = s - prod
    exact = ((prod - (s - bb)) + (p1.astype(np.float64) - bb)) == 0          # TwoSum error term
    fused = inter / (s.astype(np.float32) - inter)
    return sep, fused, exact


def wh_iou_boundary_cases(anchors, ny, nx, iou_t=0.2, n_h=400, span=48, seed=0):
    """Normalised target sizes (w, h) whose fp32 wh_iou against one anchor equals float32(iou_t) or lies one ulp either
    side of it, in the separately rounded or in the fused form.  Targets inside the anchor (gw < aw, gh < ah) have
    iou = gw * gh / (aw * ah): for n_h heights, w is scanned over +-span ulps around that solution.
    Returns a dict of arrays: a, w, h, sep, fused (the two IoUs), and the threshold as float32."""
    t32 = _f32(iou_t)
    near = np.array([np.nextafter(t32, np.float32(0)), t32, np.nextafter(t32, np.float32(1))], dtype=np.float32)
    rs = np.random.RandomState(seed)
    out = {k: [] for k in ("a", "w", "h", "sep", "fused")}
    nx32, ny32 = _f32(nx), _f32(ny)
    for a, (aw, ah) in enumerate(np.asarray(anchors, dtype=np.float32)):
        gh_want = rs.uniform(0.3, 0.95, n_h) * float(ah)
        h = (gh_want / float(ny)).astype(np.float32)
        gh = h * ny32
        w0 = (float(iou_t) * float(aw) * float(ah) / gh.astype(np.float64) / nx).astype(np.float32)
        steps = np.arange(-span, span + 1)
        w = w0[:, None].view(np.int32) + steps[None, :].astype(np.int32)
        w = w.view(np.float32)
        hh = np.broadcast_to(h[:, None], w.shape)
        gw = w * nx32
        ghh = hh * ny32
        sep, fused, exact = wh_iou_forms(aw, ah, gw, ghh)
        keep = exact & (gw < aw) & (np.isin(sep, near) | np.isin(fused, near))
        out["a"].append(np.full(int(keep.sum()), a))
        out["w"].append(w[keep])
        out["h"].append(hh[keep])
        out["sep"].append(sep[keep])
        out["fused"].append(fused[keep])
    res = {k: np.concatenate(v) for k, v in out.items()}
    res["iou_t"] = t32
    return res


def f32_preimage(target, n):
    """A float32 v with float32(v * n) == target (a normalised coordinate that lands exactly on a grid value), or None."""
    v0 = np.float32(np.float64(target) / n)
    for d in range(-4, 5):
        v = (np.array([v0]).view(np.int32) + d).view(np.float32)[0]
        if v * np.float32(n) == np.float32(target):
            return v
    return None


# ---------------------------------------------------------------------------------------------------------------------
# reference: fp32 assignment (live, the reference's arithmetic) + float64 loss
# ---------------------------------------------------------------------------------------------------------------------
def ref_assign(targets, anchor_vec, B, ny, nx, iou_t):
    """build_targets for one head in fp32 on the CPU -> (b, a, gj, gi, tbox, tcls), with the candidates that the
    reference would index out of range (image outside the batch, cell off the grid) dropped."""
    shape = types.SimpleNamespace(shape=(B, anchor_vec.shape[0], ny, nx, 1))
    tcls, tbox, ind, _ = orc.build_targets([shape], targets.float(), [anchor_vec.float()], iou_t)
    b, a, gj, gi = ind[0]
    a = torch.as_tensor(a, dtype=torch.long)                              # a python list when there are no targets
    ok = (b >= 0) & (b < B) & (gi >= 0) & (gi < nx) & (gj >= 0) & (gj < ny)
    return b[ok], a[ok], gj[ok], gi[ok], tbox[0][ok], tcls[0][ok]


def _crit(x, y, pw, gamma):
    """BCEWithLogits(pos_weight, reduction='none'), focal-modulated when gamma > 0 (utils.py:333-360), summed."""
    l = F.binary_cross_entropy_with_logits(x, y, pos_weight=torch.tensor([pw], dtype=x.dtype), reduction='none')
    if gamma > 0:
        s = torch.sigmoid(x)
        p_t = y * s + (1 - y) * (1 - s)
        l = l * (y * 0.25 + (1 - y) * 0.75) * (1.0 - p_t) ** gamma
    return l.sum()


def ref_loss(p, assign, anchor_vec, hyp, gamma, gr=1.0):
    """One head of compute_loss in float64 -> (out4 [sum(1-giou), nb, sum cls, sum obj], dp, tobj), with
    dp = d(w_box * box / nb + w_obj * obj / cells + w_cls * cls / (nb * nc)) / dp, the kernel's gradient."""
    b, a, gj, gi, tbox, tcls = assign
    B, na, ny, nx, no = p.shape
    nc = no - 5
    x = p.detach().double().requires_grad_(True)
    nb = int(b.numel())
    tobj = torch.zeros(B, na, ny, nx, dtype=torch.float64)
    box = cls = torch.zeros((), dtype=torch.float64)
    if nb:
        ps = x[b, a, gj, gi]
        pwh = torch.exp(ps[:, 2:4]).clamp(max=1E3) * anchor_vec.double()[a]
        giou = orc.giou_xywh(torch.cat((torch.sigmoid(ps[:, 0:2]), pwh), 1).t(), tbox.double())
        box = (1.0 - giou).sum()
        # tobj[b, a, gj, gi] = ... (utils.py:407).  torch leaves the winner of duplicate indices in index_put undefined,
        # and the CPU kernel does not keep list order once it runs in parallel (thousands of targets); the rule pinned
        # here is the one a sequential index_put gives and the kernel implements: the highest list position wins.
        cell = ((b * na + a) * ny + gj) * nx + gi
        win = torch.full((tobj.numel(),), -1, dtype=torch.long).scatter_reduce(0, cell, torch.arange(nb), "amax")
        hit = (win >= 0).nonzero().squeeze(1)
        tobj.view(-1)[hit] = (1.0 - gr) + gr * giou.detach()[win[hit]].clamp(0)
        if nc > 1:
            t = torch.zeros_like(ps[:, 5:])
            t[range(nb), tcls] = 1.0
            cls = _crit(ps[:, 5:], t, hyp['cls_pw'], gamma)
    obj = _crit(x[..., 4], tobj, hyp['obj_pw'], gamma)
    cells = B * na * ny * nx
    total = hyp['obj'] * obj / cells
    if nb:
        total = total + hyp['giou'] * box / nb
        if nc > 1:
            total = total + hyp['cls'] * cls / (nb * nc)
    total.backward()
    out4 = torch.tensor([float(box.detach()), nb, float(cls.detach()), float(obj.detach())], dtype=torch.float64)
    return out4, x.grad, tobj


def run_loss(p, targets, anchor_vec, hyp, gamma, want_grad=True):
    from b200yolo import ops
    nc = p.shape[-1] - 5
    out4, dp = ops.yolo_loss_layer(p.cuda(), targets.cuda(), anchor_vec.cuda(), hyp['iou_t'], 1.0, hyp['cls_pw'],
                                   hyp['obj_pw'], hyp['giou'], hyp['obj'], hyp['cls'] if nc > 1 else 0.0,
                                   want_grad=want_grad, fl_gamma=gamma)
    return out4.cpu(), (dp.cpu() if dp is not None else None)


def check_head(p, targets, anchor_vec, hyp, gamma, tag, check_tobj=True):
    """kernel vs reference on one head; returns (max item rel err, max dp err / max|dp_ref|)"""
    from b200yolo import ops
    B, na, ny, nx, no = p.shape
    assign = ref_assign(targets, anchor_vec, B, ny, nx, hyp['iou_t'])
    # build_targets: rows, order, tbox bit-exact
    idx, tbox, tcls = ops.build_targets_layer(targets.cuda(), anchor_vec.cuda(), B, ny, nx, hyp['iou_t'])
    want_idx = torch.stack(assign[:4])
    assert idx.shape == want_idx.shape, "%s: build_targets count %d vs %d" % (tag, idx.shape[1], want_idx.shape[1])
    assert torch.equal(idx.cpu(), want_idx), "%s: build_targets indices" % tag
    assert torch.equal(tcls.cpu(), assign[5]), "%s: build_targets classes" % tag
    assert torch.equal(tbox.cpu().view(torch.int32), assign[4].contiguous().view(torch.int32)), "%s: tbox bits" % tag
    # the loss
    out4, dp = run_loss(p, targets, anchor_vec, hyp, gamma)
    r4, rdp, tobj = ref_loss(p, assign, anchor_vec, hyp, gamma)
    assert int(out4[1]) == int(r4[1]) == want_idx.shape[1], "%s: nb %d vs %d" % (tag, int(out4[1]), int(r4[1]))
    if no == 6:
        assert float(out4[2]) == 0.0
    rel = 0.0
    for q in (0, 2, 3):
        ref = float(r4[q])
        err = abs(float(out4[q]) - ref)
        assert err <= 1e-5 * abs(ref), "%s: item %d: %r vs %r" % (tag, q, float(out4[q]), ref)
        rel = max(rel, err / abs(ref) if ref else 0.0)
    assert torch.isfinite(dp).all(), tag
    d = (dp.double() - rdp).abs().max().item()
    scale = rdp.abs().max().item()
    assert d <= 1e-5 * scale + 1e-7, "%s: dp err %.3g vs max|dp_ref| %.3g" % (tag, d, scale)
    if check_tobj and gamma == 0 and hyp['obj_pw'] == 1.0:
        # objectness gradient of plain BCE is (sigmoid(x) - tobj) * w_obj / cells: recover the kernel's tobj and
        # compare it with the reference's, so a wrong duplicate-cell winner fails even where dp is small
        cells = B * na * ny * nx
        got_tobj = torch.sigmoid(p[..., 4].double()) - dp[..., 4].double() * cells / hyp['obj']
        terr = (got_tobj - tobj).abs().max().item()
        assert terr < 1e-4, "%s: tobj err %.3g" % (tag, terr)
    return rel, d / max(scale, 1e-30), int(r4[1])


def _targets(rs, B, nt, nc, share=0.5, fine=80):
    """nt targets over B images; a fraction `share` copy the cell (image, x, y on a fine x fine grid) of a random earlier
    target, with new sizes and classes, and everything is shuffled: duplicates sit at distant list positions."""
    t = np.zeros((nt, 6), dtype=np.float32)
    if nt == 0:
        return torch.from_numpy(t)
    t[:, 0] = rs.randint(0, B, nt)
    t[:, 1] = rs.randint(0, nc, nt)
    t[:, 2:4] = rs.uniform(0.0, 1.0, (nt, 2))
    t[:, 4:6] = np.exp(rs.uniform(np.log(0.01), np.log(0.7), (nt, 2)))
    n_dup = int(nt * share)
    if n_dup and nt > 1:
        src = rs.randint(0, nt - n_dup, n_dup)
        dst = np.arange(nt - n_dup, nt)
        cell = np.floor(t[src, 2:4] * fine)
        t[dst, 0] = t[src, 0]
        t[dst, 2:4] = ((cell + rs.uniform(0.05, 0.95, (n_dup, 2))) / fine).astype(np.float32)
    t = t[rs.permutation(nt)]
    return torch.from_numpy(np.ascontiguousarray(t))


# ---------------------------------------------------------------------------------------------------------------------
# host: the boundary constructor against the reference's torch expressions
# ---------------------------------------------------------------------------------------------------------------------
def test_boundary_constructor_matches_reference_expressions():
    """wh_iou_boundary_cases builds what it claims: its 'sep' IoU is the reference's wh_iou on targets * gain in torch
    float32, bit for bit; its 'fused' IoU is the exactly rounded FMA form; every case sits within an ulp of iou_t; and
    for the stock yolov3 anchors at iou_t = 0.2 some cases are decided differently by the two forms."""
    from fractions import Fraction
    total_flips = 0
    for anchors_px, stride, n in zip(V3, (8, 16, 32), (80, 40, 20)):
        av = _av(anchors_px, stride)
        cases = wh_iou_boundary_cases(av.numpy(), n, n)
        assert len(cases["a"]) > 0
        t32 = cases["iou_t"]
        targets = torch.zeros(len(cases["a"]), 6)
        targets[:, 4] = torch.from_numpy(cases["w"])
        targets[:, 5] = torch.from_numpy(cases["h"])
        gain = torch.ones(6)
        gain[2:] = torch.tensor([n, n, n, n]).float()
        gwh = (targets * gain)[:, 4:6]
        iou = orc.wh_iou(av, gwh)                                         # [na, nt], the reference's expression
        a = torch.from_numpy(cases["a"])
        ref = iou[a, torch.arange(len(a))]
        assert torch.equal(ref, torch.from_numpy(cases["sep"])), "constructor's separately rounded IoU != torch"
        ulp = np.abs(cases["sep"].view(np.int32).astype(np.int64) - np.array([t32]).view(np.int32)[0])
        ulf = np.abs(cases["fused"].view(np.int32).astype(np.int64) - np.array([t32]).view(np.int32)[0])
        assert (np.minimum(ulp, ulf) <= 1).all()
        # the fused form against exact rational arithmetic, rounded once to float32 (round to nearest even)
        for k in range(0, len(a), max(1, len(a) // 50)):
            aw, ah = (float(v) for v in av[int(a[k])])
            gw, gh = float(gwh[k, 0]), float(gwh[k, 1])
            s = Fraction(gw) * Fraction(gh) + Fraction(float(np.float32(aw) * np.float32(ah)))
            lo = np.float32(float(s))
            cands = [lo, np.nextafter(lo, np.float32(-np.inf)), np.nextafter(lo, np.float32(np.inf))]
            best = min(cands, key=lambda c: (abs(Fraction(float(c)) - s), int(np.array([c]).view(np.int32)[0]) & 1))
            inter = np.float32(min(aw, gw)) * np.float32(min(ah, gh))
            assert np.float32(inter / (best - inter)) == cases["fused"][k]
        flips = int(((cases["sep"] > t32) != (cases["fused"] > t32)).sum())
        total_flips += flips
        assert int((ref > 0.2).sum()) == int((cases["sep"] > t32).sum())    # torch compares against float32(0.2)
    assert total_flips > 0, "no candidate decided differently by the fused and the separately rounded wh_iou"


def test_cell_preimages_land_on_the_grid():
    for n in (13, 20, 40, 80):
        for k in (0, 1, n // 2, n - 1):
            v = f32_preimage(k, n)
            assert v is not None and v * np.float32(n) == np.float32(k)
            assert int(torch.tensor([v]) * torch.tensor([float(n)])) == k


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,per_image,seed", [(8, 0, 0), (8, 40, 1), (16, 190, 2)], ids=["nt0", "nt320", "nt3040"])
def test_loss_at_training_scale(B, per_image, seed):
    """yolov4's three heads at 640^2 (80, 40, 20 grids); up to ~3000 targets, half of them sharing a cell with a distant
    list entry, so that na * nt is far above one 1024-thread chunk and the duplicate-cell winners race across CTAs."""
    rs = np.random.RandomState(seed)
    nt = B * per_image
    t = _targets(rs, B, nt, 80)
    g = torch.Generator().manual_seed(seed)
    worst = [0.0, 0.0]
    for anchors_px, stride in zip(V4, V4_STRIDES):
        n = 640 // stride
        p = torch.randn(B, 3, n, n, 85, generator=g) * 1.5
        rel, drel, nb = check_head(p, t, _av(anchors_px, stride), HYP, 0.0, "v4/%d nt=%d" % (n, nt))
        worst = [max(worst[0], rel), max(worst[1], drel)]
        print("\n[scale] grid %d nt %d: nb %d, item rel err %.3g, dp err / max %.3g" % (n, nt, nb, rel, drel))
    print("[scale] nt %d: largest item rel err %.3g, largest dp err / max|dp| %.3g" % (nt, worst[0], worst[1]))


HEAD_CASES = [
    # (id, anchors (grid units), no, ny, nx, gamma)
    ("v2-na5-13x20", V2, 85, 13, 20, 0.0),
    ("nc1-20x13", _av(V3[1], 16).tolist(), 6, 20, 13, 0.0),
    ("nc100-13x20-g1.5", _av(V3[2], 32).tolist(), 105, 13, 20, 1.5),
    ("nc2-26x40", _av(V3[0], 8).tolist(), 7, 26, 40, 0.0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", HEAD_CASES, ids=[c[0] for c in HEAD_CASES])
def test_head_shapes_and_non_square_grids(case):
    """na = 5 (yolov2), nc = 1 (no class term, out4[2] == 0), nc = 100 and nc = 2, on grids with ny != nx, so that a
    swapped nx / ny or gi / gj fails."""
    tag, anchors, no, ny, nx, gamma = case
    av = torch.tensor(anchors, dtype=torch.float32)
    rs = np.random.RandomState(7)
    B = 4
    t = _targets(rs, B, 300, no - 5, fine=max(ny, nx))
    # a band of targets far off-centre in x only or in y only: a transposed grid puts them in different cells
    t[:40, 2] = torch.from_numpy(rs.uniform(0.0, 0.2, 40).astype(np.float32))
    t[:40, 3] = torch.from_numpy(rs.uniform(0.8, 1.0, 40).astype(np.float32))
    hyp = dict(HYP, cls=HYP['cls'] * (no - 5) / 80.0)
    p = torch.randn(B, av.shape[0], ny, nx, no, generator=torch.Generator().manual_seed(3))
    rel, drel, nb = check_head(p, t, av, hyp, gamma, tag)
    print("\n[%s] nb %d, item rel err %.3g, dp err / max %.3g" % (tag, nb, rel, drel))


def _edge_head(gamma):
    """One yolov3 stride-16 head on a 13 x 20 grid with: targets on cell boundaries (x * nx an exact integer, x = 0),
    a prediction equal to its target box (min / max selectors tie), width / height logits past the exp clamp, and
    objectness / class logits of +-30."""
    av = _av(V3[1], 16)
    B, na, ny, nx, no = 2, 3, 13, 20, 85
    rs = np.random.RandomState(11)
    rows = []
    for k in (0, 1, 7, nx - 1):                                    # x * nx == k exactly
        for kk in (0, 5, ny - 1):
            x, y = f32_preimage(k, nx), f32_preimage(kk, ny)
            rows.append([k % B, k % 80, float(x), float(y), 0.3, 0.25])
    rows.append([1, 3, 0.0, 0.0, 0.5, 0.4])
    # prediction == target: logits 0 give sigmoid 0.5 and exp 1 in every precision, so the target is (k + 0.5, k' + 0.5)
    # with width / height equal to anchor 1
    tie_cell = (0, 1, 6, 11)                                      # (b, a, gj, gi)
    aw, ah = (np.float32(v) for v in av[1])
    rows.append([0, 9] + [float(f32_preimage(v, n)) for v, n in ((11.5, nx), (6.5, ny), (aw, nx), (ah, ny))])
    # saturated width / height logits on a cell of its own
    sat_cell = (1, 2, 2, 3)
    rows.append([1, 4, float(f32_preimage(3.5, nx)), float(f32_preimage(2.5, ny)), 0.25, 0.6])
    t = torch.tensor(np.asarray(rows, dtype=np.float32))
    t = torch.cat([t, _targets(rs, B, 60, 80, fine=nx)])
    p = torch.randn(B, na, ny, nx, no, generator=torch.Generator().manual_seed(5))
    p[tie_cell][:4] = 0.0
    p[sat_cell][2:4] = torch.tensor([8.0, 9.5])                   # exp > 1e3: clamped, no gradient
    sat = torch.rand(B, na, ny, nx, no, generator=torch.Generator().manual_seed(6)) < 0.3
    sat[..., :4] = False
    p[sat] = torch.where(torch.rand(int(sat.sum()), generator=torch.Generator().manual_seed(8)) < 0.5, 30.0, -30.0)
    return p, t, av, tie_cell, sat_cell


@pytest.mark.gpu
@pytest.mark.parametrize("gamma", [0.0, 0.5, 1.5])
def test_decision_edges(gamma):
    p, t, av, tie_cell, sat_cell = _edge_head(gamma)
    rel, drel, nb = check_head(p, t, av, HYP, gamma, "edges g%.1f" % gamma, check_tobj=False)
    out4, dp = run_loss(p, t, av, HYP, gamma)
    assert torch.equal(dp[sat_cell][2:4], torch.zeros(2)), "clamped exp must carry no gradient"
    assert torch.isfinite(dp).all()
    print("\n[edges gamma %.1f] nb %d, item rel err %.3g, dp err / max %.3g, tie-cell dp %s"
          % (gamma, nb, rel, drel, dp[tie_cell][:4].tolist()))


@pytest.mark.gpu
def test_wh_iou_threshold_candidates():
    """Targets whose fp32 wh_iou against an anchor is float32(iou_t) or one ulp either side of it.  Where the separately
    rounded IoU and an FMA-contracted one fall on different sides of iou_t, only the former is the reference."""
    B = 2
    n_cases = n_flips = 0
    for anchors_px, stride, n in zip(V3, (8, 16, 32), (80, 40, 20)):
        av = _av(anchors_px, stride)
        cases = wh_iou_boundary_cases(av.numpy(), n, n)
        t32 = cases["iou_t"]
        flips = (cases["sep"] > t32) != (cases["fused"] > t32)
        m = len(cases["a"])
        n_cases += m
        n_flips += int(flips.sum())
        rs = np.random.RandomState(n)
        t = np.zeros((m, 6), dtype=np.float32)
        t[:, 0] = rs.randint(0, B, m)
        t[:, 1] = rs.randint(0, 80, m)
        t[:, 2:4] = rs.uniform(0, 1, (m, 2))
        t[:, 4], t[:, 5] = cases["w"], cases["h"]
        t = torch.from_numpy(t)
        p = torch.randn(B, 3, n, n, 85, generator=torch.Generator().manual_seed(n))
        check_head(p, t, av, HYP, 0.0, "threshold grid %d" % n, check_tobj=False)
    print("\n[threshold] %d boundary candidates built, %d decided differently by the fused and the separately rounded "
          "wh_iou" % (n_cases, n_flips))
    assert n_flips > 0


@pytest.mark.gpu
def test_out_of_range_candidates_are_dropped():
    """x == 1.0 / y == 1.0 (cell index nx / ny after truncation), and image indices -1 and B: both kernels drop them."""
    av = _av(V3[2], 32)
    B, ny, nx = 2, 13, 20
    bad = torch.tensor([[0, 1, 1.0, 0.5, 0.3, 0.3], [1, 2, 0.5, 1.0, 0.3, 0.3], [2, 3, 0.5, 0.5, 0.3, 0.3],
                        [-1, 4, 0.5, 0.5, 0.3, 0.3]], dtype=torch.float32)
    good = torch.tensor([[0, 5, 0.4, 0.6, 0.3, 0.3], [1, 6, 0.999, 0.999, 0.3, 0.3]], dtype=torch.float32)
    t = torch.cat([bad[:2], good[:1], bad[2:], good[1:]])
    p = torch.randn(B, 3, ny, nx, 85, generator=torch.Generator().manual_seed(1))
    check_head(p, t, av, HYP, 0.0, "out of range")
    _, _, nb_good = check_head(p, good, av, HYP, 0.0, "in range")
    out4, _ = run_loss(p, t, av, HYP, 0.0)
    assert int(out4[1]) == nb_good > 0


@pytest.mark.gpu
def test_eval_launch_and_workspace_reuse():
    """want_grad=False (test.py's eval loss) gives the gradient launch's out4; a workspace reused across launches with
    different targets is reset (winner / nb), so the same targets give the same nb and the same objectness gradient."""
    from b200yolo import ops
    from b200yolo.lib import call, ptr, raw, stream_ptr
    av = _av(V4[1], 16).cuda()
    B, na, ny, nx, no = 8, 3, 40, 40, 85
    rs = np.random.RandomState(4)
    ta, tb = _targets(rs, B, 600, 80).cuda(), _targets(rs, B, 900, 80).cuda()
    p = torch.randn(B, na, ny, nx, no, generator=torch.Generator().manual_seed(2)).cuda()
    h = HYP
    o_g, dp_g = run_loss(p, ta, av, h, 0.0)
    o_e, dp_e = run_loss(p, ta, av, h, 0.0, want_grad=False)
    assert dp_e is None
    assert float(o_e[1]) == float(o_g[1])
    torch.testing.assert_close(o_e, o_g, rtol=1e-6, atol=0)
    ws = torch.empty(raw().b2y_yolo_loss_workspace_bytes(B, na, ny, nx, 900), dtype=torch.uint8, device="cuda")
    out4 = torch.empty(4, device="cuda")

    def launch(t, dp):
        call("b2y_yolo_loss", ptr(p), ptr(t), int(t.shape[0]), ptr(av), B, na, no, ny, nx, h['iou_t'], 1.0,
             h['cls_pw'], h['obj_pw'], h['giou'], h['obj'], h['cls'], 0.0, ptr(out4), ptr(dp), ptr(ws), stream_ptr())
        return out4.clone().cpu()

    runs = []
    for t in (ta, tb, ta, tb, ta):
        dp = torch.empty_like(p)
        runs.append((launch(t, dp), dp.cpu()))
    for k in (2, 4):
        assert float(runs[k][0][1]) == float(runs[0][0][1]) == float(o_g[1])
        assert torch.equal(runs[k][1][..., 4], runs[0][1][..., 4]), "objectness gradient depends on the previous launch"
        torch.testing.assert_close(runs[k][0], runs[0][0], rtol=1e-6, atol=0)
    assert float(runs[1][0][1]) == float(runs[3][0][1])
    assert torch.equal(runs[0][1][..., 4], dp_g[..., 4])


@pytest.mark.gpu
@pytest.mark.parametrize("na,nt", [(3, 341), (1, 1024), (5, 205), (3, 3001)], ids=["1023", "1024", "1025", "9003"])
def test_build_targets_chunk_boundaries(na, nt):
    """The one-CTA ordered compaction at na * nt = 1023, 1024, 1025 and ~9000 (1024-thread chunks): row order
    (anchor-major, target-minor), idx, tbox and tcls exactly as the reference's build_targets."""
    from b200yolo import ops
    av = torch.tensor([[3.0, 3.0], [3.5, 2.8], [2.8, 3.6], [3.2, 3.3], [2.9, 2.9]])[:na]
    B, ny, nx = 4, 20, 20
    rs = np.random.RandomState(na * nt)
    t = _targets(rs, B, nt, 80)
    # four in five targets match every anchor, so that the emitted rows run across the chunk edges
    most = torch.from_numpy(rs.uniform(0, 1, nt) < 0.8)
    t[most, 4] = 3.1 / nx
    t[most, 5] = 3.1 / ny
    want = ref_assign(t, av, B, ny, nx, HYP['iou_t'])
    idx, tbox, tcls = ops.build_targets_layer(t.cuda(), av.cuda(), B, ny, nx, HYP['iou_t'])
    assert idx.shape[1] == want[0].numel()
    assert torch.equal(idx.cpu(), torch.stack(want[:4]))
    assert torch.equal(tbox.cpu().view(torch.int32), want[4].contiguous().view(torch.int32))
    assert torch.equal(tcls.cpu(), want[5])
    print("\n[build_targets] na*nt %d: %d rows" % (na * nt, idx.shape[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("gdt", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("na,no,pitch", [(5, 85, 432), (3, 105, 320)], ids=["432", "320"])
def test_yolo_grad_to_raw_wide_heads(na, no, pitch, gdt):
    """dp [B, na, ny, nx, no] -> d raw [B, ny, nx, pitch] times scale * (device scale), one rounding; the pad columns
    na * no .. pitch are written as exact zeros over a buffer that held garbage."""
    from b200yolo import ops
    from b200yolo.lib import call, ptr, stream_ptr
    B, ny, nx = 2, 13, 20
    dp = torch.randn(B, na, ny, nx, no, generator=torch.Generator().manual_seed(na))
    raw = torch.full((B, ny, nx, pitch), 7.0, dtype=gdt, device="cuda")
    sc = torch.tensor([3.0], device="cuda")
    call("b2y_yolo_grad_to_raw", ptr(dp.cuda()), ptr(raw), pitch, B, na, no, ny, nx, 0.5, ptr(sc), ops._gdt(raw),
         stream_ptr())
    want = (dp.permute(0, 2, 3, 1, 4).reshape(B, ny, nx, na * no) * 1.5).to(gdt)
    got = raw.cpu()
    assert torch.equal(got[..., :na * no], want)
    assert torch.equal(got[..., na * no:], torch.zeros(B, ny, nx, pitch - na * no, dtype=gdt))


@pytest.mark.gpu
def test_yolo_decode_run_kernel_na5():
    """b2y_yolo_decode with na * no = 425 > 256 (the run-per-warp kernel yolov2 takes) on a 13 x 20 grid, raw pitch
    432: p bit-exact, grid indices exact, values as YOLOLayer.forward (models.py:401-437)."""
    from b200yolo import ops
    g = torch.Generator().manual_seed(6)
    B, na, no, ny, nx, stride = 2, 5, 85, 13, 20, 32.0
    anchors = torch.tensor(V2) * stride
    raw_nchw = torch.randn(B, na * no, ny, nx, generator=g)
    p = raw_nchw.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
    yv, xv = torch.meshgrid([torch.arange(ny), torch.arange(nx)], indexing="ij")
    grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2).float()
    io = p.clone()
    io[..., :2] = torch.sigmoid(io[..., :2]) + grid
    io[..., 2:4] = torch.exp(io[..., 2:4]) * (anchors / stride).view(1, na, 1, 1, 2)
    io[..., :4] *= stride
    torch.sigmoid_(io[..., 4:])
    raw = torch.full((B, ny, nx, 432), float("nan"), dtype=torch.float32, device="cuda")
    raw[..., :na * no] = raw_nchw.permute(0, 2, 3, 1).cuda()
    total = na * ny * nx + 5
    iobuf = torch.zeros(B, total, no, device="cuda")
    _, pg = ops.yolo_decode(raw, na, no, anchors.cuda(), stride, io=iobuf, row_offset=5)
    torch.cuda.synchronize()
    assert torch.equal(pg.cpu(), p), "p (permuted raw) must be bit exact"
    got = iobuf[:, 5:].cpu().view(B, na, ny, nx, no)
    cell = torch.round(got[..., :2] / stride - torch.sigmoid(p[..., :2]))
    assert torch.equal(cell, grid.expand_as(cell)), "grid indices must be exact"
    torch.testing.assert_close(got, io, rtol=1e-5, atol=1e-6)
    assert float(iobuf[:, :5].abs().max()) == 0
