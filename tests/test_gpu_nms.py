"""GPU: detection post-processing on the device (SURVEY section 8 row f1): utils.utils.non_max_suppression and the
true-positive matching of test.py, csrc/nms.cu through the C ABI, against

  * the reference's own outputs (tests/golden/map_case.npz, oracle/gen_golden_map.py: its non_max_suppression +
    clip_coords + matching loop on a yolov3-tiny prediction), and
  * oracle/metrics_oracle.py (pinned to the same fixture) on synthetic predictions that exercise what the fixture does
    not: score ties, rows rejected by the size / confidence / finite filters, best-class and class-agnostic modes, the
    `classes=` filter, images without candidates, n >= 3000 (no merge), more than 512 kept boxes (several tiles of the
    kept list) and chunk boundaries of the greedy kernel.

Bar: kept set, order, scores and classes bit-exact; boxes bit-exact where the reference does not merge, 1e-5 relative
where it does (its torch.mm sums in a different order); TP matrices bit-exact."""
import numpy as np
import pytest
import torch

from helpers import golden
from oracle import metrics_oracle as mo

pytestmark = pytest.mark.gpu

MERGE_RTOL = 1e-5       # the test prints the measured maxima


def synth_predictions(B, R, nc, seed, n_obj=30, per_obj=12, bg_pass=0.02, small_boxes=0):
    """[B, R, 5 + nc] predictions with the statistics of a trained detector: most rows fail the confidence filter,
    objects are clusters of jittered boxes with one or two strong classes, scores come from a coarse grid (ties)."""
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(B, R, 5 + nc)
    p[..., 0] = torch.rand(B, R, generator=g) * 640
    p[..., 1] = torch.rand(B, R, generator=g) * 640
    p[..., 2:4] = torch.exp(torch.rand(B, R, 2, generator=g) * 4.0 + 1.0)          # 2.7 .. 148 px
    p[..., 4] = torch.rand(B, R, generator=g) * 0.04
    p[..., 5:] = torch.rand(B, R, nc, generator=g) * 0.2
    passing = torch.rand(B, R, generator=g) < bg_pass
    p[..., 4] = torch.where(passing, torch.rand(B, R, generator=g) * 0.6 + 0.2, p[..., 4])
    levels = torch.tensor([0.25, 0.5, 0.75, 1.0])
    for b in range(B):
        rows = torch.randperm(R, generator=g)
        k = 0
        for _ in range(n_obj):
            c = torch.rand(2, generator=g) * 500 + 70
            wh = torch.exp(torch.rand(2, generator=g) * 2.5 + 2.5)                  # 12 .. 150 px
            cls = int(torch.randint(0, nc, (1,), generator=g))
            for _ in range(per_obj):
                if k >= R:
                    break
                r = int(rows[k]); k += 1
                p[b, r, 0:2] = c + torch.randn(2, generator=g) * 0.06 * wh
                p[b, r, 2:4] = wh * torch.exp(torch.randn(2, generator=g) * 0.08)
                p[b, r, 4] = levels[int(torch.randint(1, 4, (1,), generator=g))]
                p[b, r, 5:] = torch.rand(nc, generator=g) * 0.05
                p[b, r, 5 + cls] = levels[int(torch.randint(0, 4, (1,), generator=g))]
                if nc > 1 and torch.rand(1, generator=g) < 0.3:
                    p[b, r, 5 + (cls + 1) % nc] = levels[int(torch.randint(0, 3, (1,), generator=g))]
        for _ in range(small_boxes):                                                 # many disjoint kept boxes
            if k >= R:
                break
            r = int(rows[k]); k += 1
            p[b, r, 0:2] = torch.rand(2, generator=g) * 620 + 10
            p[b, r, 2:4] = torch.rand(2, generator=g) * 6 + 4
            p[b, r, 4] = 0.9
            p[b, r, 5:] = 0.0
            p[b, r, 5 + int(torch.randint(0, nc, (1,), generator=g))] = float(torch.rand(1, generator=g)) * 0.5 + 0.4
    return p


def _compare(got, want, tag):
    """got: list from the device path, want: list from the oracle / reference.  Returns the worst merged-box error."""
    assert len(got) == len(want)
    worst = 0.0
    for b, (g, w) in enumerate(zip(got, want)):
        if w is None:
            assert g is None, "%s image %d: reference has no detections, device path has %d" % (tag, b, len(g))
            continue
        assert g is not None, "%s image %d: device path lost all %d detections" % (tag, b, len(w))
        g = g.cpu()
        assert g.shape == w.shape, "%s image %d: kept %d vs reference %d" % (tag, b, g.shape[0], w.shape[0])
        # scores and classes (and therefore the kept set and its order) bit-exact
        assert torch.equal(g[:, 4], w[:, 4]), "%s image %d: scores differ" % (tag, b)
        assert torch.equal(g[:, 5], w[:, 5]), "%s image %d: classes differ" % (tag, b)
        err = ((g[:, :4] - w[:, :4]).abs() / w[:, :4].abs().clamp(min=1.0)).max().item()
        worst = max(worst, err)
    return worst


def test_nms_and_matching_reproduce_the_reference_fixture():
    """The reference's own non_max_suppression / clip_coords / matching outputs on a yolov3-tiny prediction."""
    from b200yolo import detect
    g = golden("map_case")
    inf_out = torch.from_numpy(g["inf_out"])
    S = int(g["size"])
    packed = detect.nms_packed(inf_out.cuda(), conf_thres=0.3, iou_thres=0.6)       # oracle/gen_golden_map.py: CONF, IOU
    B = inf_out.shape[0]
    labels = [torch.from_numpy(g["labels%d" % i]) for i in range(B)]
    tcls = torch.cat([lab[:, 0] for lab in labels])
    tbox = torch.cat([lab[:, 1:5] for lab in labels])
    lab_off = torch.tensor([0] + list(np.cumsum([lab.shape[0] for lab in labels])), dtype=torch.int32)
    correct = detect.match_labels(packed, tcls, tbox, lab_off, torch.linspace(0.5, 0.95, 10), S, S)
    want = [torch.from_numpy(g["det%d" % i]) for i in range(B)]                      # clipped, like `packed.det` now
    worst = _compare(packed.to_list(), want, "fixture")
    print("\n[nms fixture] detections %s, worst merged-box error %.3g (gate %.0e)" % (packed.counts, worst, MERGE_RTOL))
    assert worst <= MERGE_RTOL
    for i in range(B):
        assert np.array_equal(correct[i].cpu().numpy(), g["correct%d" % i]), "TP matrix of image %d differs" % i


CASES = [
    # name, B, R, nc, kwargs of synth_predictions, nms kwargs
    ("multi_label", 3, 4000, 80, dict(n_obj=40, per_obj=14), dict(conf_thres=0.1, iou_thres=0.6)),
    ("low_conf_many_candidates", 2, 6000, 20, dict(n_obj=60, per_obj=20, bg_pass=0.1),
     dict(conf_thres=0.05, iou_thres=0.6)),                                          # n >= 3000: no merge, exact boxes
    ("many_kept", 2, 5000, 80, dict(n_obj=10, per_obj=8, small_boxes=1500), dict(conf_thres=0.3, iou_thres=0.5)),
    ("best_class", 2, 3000, 80, dict(n_obj=30, per_obj=10), dict(conf_thres=0.1, iou_thres=0.6, multi_label=False)),
    ("agnostic", 2, 3000, 10, dict(n_obj=30, per_obj=10), dict(conf_thres=0.1, iou_thres=0.45, agnostic=True)),
    ("class_filter", 2, 3000, 10, dict(n_obj=30, per_obj=10), dict(conf_thres=0.1, iou_thres=0.6, classes=[1, 4, 7])),
    ("single_class", 2, 2000, 1, dict(n_obj=20, per_obj=10), dict(conf_thres=0.1, iou_thres=0.6)),
    ("chunk_edges", 4, 1500, 4, dict(n_obj=43, per_obj=12, bg_pass=0.0), dict(conf_thres=0.05, iou_thres=0.6)),
]


@pytest.mark.parametrize("name,B,R,nc,skw,nkw", CASES, ids=[c[0] for c in CASES])
def test_nms_matches_oracle(name, B, R, nc, skw, nkw):
    from b200yolo import detect
    pred = synth_predictions(B, R, nc, seed=len(name) * 7 + R, **skw)
    if name == "multi_label":
        pred[0, 5, 0] = float("nan")                    # non-finite box on a row that passes the filters
        pred[0, 5, 2:5] = torch.tensor([20.0, 20.0, 0.9])
        pred[0, 6, 2:5] = torch.tensor([20.0, 20.0, 0.9])
        pred[0, 6, 5 + 3] = float("inf")                # inf * obj: passes `> conf_thres`, dropped as non-finite
        pred[0, 7, 2:5] = torch.tensor([5000.0, 20.0, 0.9])       # too wide
        pred[0, 8, 2:5] = torch.tensor([2.0, 20.0, 0.9])          # width == min_wh is rejected (strict >)
        pred[2, :, 4] = 0.0                             # an image without candidates -> None
    if name == "chunk_edges":
        pred[1, :, 4] = 0.0
        pred[1, 17, :] = 0.0
        pred[1, 17, :6] = torch.tensor([100.0, 100.0, 30.0, 30.0, 0.9, 0.8])      # exactly one candidate (n == 1)
    want = mo.nms(pred.clone(), **nkw)
    got = detect.non_max_suppression(pred.cuda(), **nkw)
    worst = _compare(got, want, name)
    n_kept = [0 if w is None else w.shape[0] for w in want]
    print("\n[nms %s] kept %s, worst box error %.3g" % (name, n_kept, worst))
    if name == "low_conf_many_candidates":
        assert worst == 0.0, "n >= 3000: the reference does not merge, boxes must be bit-exact"
    assert worst <= MERGE_RTOL
    if name == "many_kept":
        assert max(n_kept) > 1024, "case must cover several tiles of the kept list"


def test_tp_matching_matches_oracle():
    """Detections of a synthetic batch against labels that are jittered copies of some of them (with duplicates, so that
    several predictions compete for one target and several targets share a best prediction)."""
    from b200yolo import detect
    B, R, nc = 3, 4000, 12
    pred = synth_predictions(B, R, nc, seed=11, n_obj=40, per_obj=10)
    pred[2, :, 4] = 0.0
    packed = detect.nms_packed(pred.cuda(), conf_thres=0.1, iou_thres=0.6)
    ref = mo.nms(pred.clone(), conf_thres=0.1, iou_thres=0.6)
    g = torch.Generator().manual_seed(5)
    labels = []
    for b in range(B):
        if ref[b] is None:
            labels.append(torch.tensor([[1.0, 10, 10, 50, 50]]))                    # labels, no detections
            continue
        d = ref[b]
        pick = torch.randperm(d.shape[0], generator=g)[: max(1, d.shape[0] // 3)]
        pick = torch.cat([pick, pick[:5]])                                          # duplicate targets
        box = d[pick, :4] + torch.randn(pick.numel(), 4, generator=g) * 3.0
        cls = d[pick, 5].clone()
        cls[::7] = (cls[::7] + 1) % nc                                              # some labels of another class
        labels.append(torch.cat([cls[:, None], box], 1))
    labels[0] = labels[0][:0]                                                       # an image without labels
    tcls = torch.cat([lab[:, 0] for lab in labels])
    tbox = torch.cat([lab[:, 1:5] for lab in labels])
    lab_off = torch.tensor([0] + list(np.cumsum([lab.shape[0] for lab in labels])), dtype=torch.int32)
    correct = detect.match_labels(packed, tcls, tbox, lab_off, mo.IOU_THRESHOLDS, 640, 640)
    dets = packed.to_list()
    n_tp = 0
    for b in range(B):
        if ref[b] is None:
            assert correct[b] is None
            continue
        d = ref[b].clone()
        mo.clip_boxes(d, 640, 640)
        # the device path clipped in place: same boxes as the oracle's (merged boxes to MERGE_RTOL)
        assert ((dets[b][:, :4].cpu() - d[:, :4]).abs() / d[:, :4].abs().clamp(min=1.0)).max().item() <= MERGE_RTOL
        want = mo.match_image(dets[b].cpu(), labels[b])                            # same boxes in: bit-exact out
        assert torch.equal(correct[b].cpu(), want), "TP matrix of image %d differs" % b
        n_tp += int(want[:, 0].sum())
    assert n_tp > 20, "degenerate case"           # measured: 41 true positives at IoU 0.5


def test_reference_entry_point_and_cpu_tensor():
    """utils.utils.non_max_suppression is the device path; CPU tensors fail loudly (no fallback)."""
    from utils import utils as my_utils
    from b200yolo import lib
    pred = synth_predictions(1, 500, 5, seed=2, n_obj=5, per_obj=6)
    out = my_utils.non_max_suppression(pred.cuda(), conf_thres=0.2, iou_thres=0.5)
    want = mo.nms(pred.clone(), conf_thres=0.2, iou_thres=0.5)
    assert _compare(out, want, "entry") <= MERGE_RTOL
    with pytest.raises(lib.B2YError):
        my_utils.non_max_suppression(pred)


def test_map_through_the_device_pipeline_matches_reference():
    """BASELINE north_star (mAP on a held batch within 1e-4 of the reference) with EVERYTHING on the device: engine forward
    in the fp32-accurate mode -> csrc/nms.cu NMS -> clip + TP matching kernel; only the AP bookkeeping (ap_per_class,
    numpy in the reference too, utils.py:162-251) runs on the host."""
    from b200yolo import detect
    from helpers import build_model, orc
    g = golden("map_case")
    S, B = int(g["size"]), g["inf_out"].shape[0]
    model = build_model("yolov3-tiny", device="cuda").eval()
    model.accurate = True
    x = orc.synth_images(B, S, S, seed=int(g["seed"]))
    with torch.no_grad():
        io, _, _ = model(x.cuda())
    packed = detect.nms_packed(io, conf_thres=0.3, iou_thres=0.6)
    labels = [torch.from_numpy(g["labels%d" % i]) for i in range(B)]
    tcls = torch.cat([lab[:, 0] for lab in labels])
    tbox = torch.cat([lab[:, 1:5] for lab in labels])
    lab_off = torch.tensor([0] + list(np.cumsum([lab.shape[0] for lab in labels])), dtype=torch.int32)
    correct = detect.match_labels(packed, tcls, tbox, lab_off, mo.IOU_THRESHOLDS, S, S)
    dets = packed.to_list()
    stats = [(correct[b].cpu().numpy(), dets[b][:, 4].cpu().numpy(), dets[b][:, 5].cpu().numpy(),
              labels[b][:, 0].numpy()) for b in range(B) if dets[b] is not None]
    cols = [np.concatenate(c, 0) for c in zip(*stats)]
    _, _, ap, _ = mo.ap_per_class(*cols)
    m50, m = float(ap[:, 0].mean()), float(ap.mean(1).mean())
    r50, r = float(g["map50"]), float(g["map"])
    print("\n[mAP, device pipeline] reference %.6f / %.6f | device %.6f / %.6f (%d detections)"
          % (r50, r, m50, m, cols[0].shape[0]))
    assert abs(m50 - r50) <= 1e-4 and abs(m - r) <= 1e-4
