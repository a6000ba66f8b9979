"""CPU: heads wider than 256 outputs and the focal loss.  The generated yolov2 cfgs against the reference's parse, the
oracle's focal branch and wide-head training steps against fixtures the reference produced (oracle/gen_golden_heads.py),
and the head widths the training plan gives every head."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from helpers import GOLD, anchor_vecs, cfg_path, golden, module_defs, orc
from oracle import focal_oracle

NC100 = None


def nc100_cfg():
    """yolov3-tiny with 100 classes: two heads of 3 * 105 = 315 filters."""
    global NC100
    from b200yolo import cfggen
    if NC100 is None:
        NC100 = os.path.join(tempfile.mkdtemp(prefix="b2y_nc100_"), "yolov3-tiny-nc100.cfg")
        with open(NC100, "w") as f:
            f.write(cfggen.cfg_text("yolov3-tiny", classes=100))
    return NC100


def _anchor_vecs_of(path, name):
    from utils.parse_config import parse_model_cfg
    ys = [d for d in parse_model_cfg(path)[1:] if d['type'] == 'yolo']
    strides = orc.yolo_strides(name, len(ys))
    return [torch.as_tensor(np.asarray(d['anchors'])[d['mask']], dtype=torch.float32) / s for d, s in zip(ys, strides)]


def _hyp(nc, gamma=0.0):
    h = dict(orc.DEFAULT_HYP)
    h['cls'] = h['cls'] * nc / 80.0
    h['fl_gamma'] = gamma
    return h


@pytest.mark.parametrize("name", ["yolov2", "yolov2-tiny"])
def test_generated_v2_cfg_equals_reference_cfg(name):
    with open(os.path.join(GOLD, "heads_cfg.json")) as f:
        ref = json.load(f)[name]
    ours = module_defs(name)
    assert len(ours) == len(ref)
    keys = ('type', 'batch_normalize', 'filters', 'size', 'stride', 'pad', 'activation', 'layers', 'from', 'mask',
            'classes', 'num')
    for a, b in zip(ours, ref):
        for k in keys:
            v = a.get(k)
            assert (v.tolist() if hasattr(v, "tolist") else v) == b.get(k), (name, k, a, b)
        if 'anchors' in b:
            assert np.array_equal(np.asarray(a['anchors']), np.asarray(b['anchors']))
    assert orc.yolo_strides(name, 1) == [32]


@pytest.mark.parametrize("case", ["g15", "g05", "sat", "dup"])
def test_oracle_focal_loss_matches_reference(case):
    g = golden("focal_case")
    if case == "dup":
        preds, t, av = [g["dup_p0"], g["dup_p1"]], g["dup_targets"], anchor_vecs("yolov3-tiny")
    else:
        pre = "sat_p" if case == "sat" else "p"
        preds, t, av = [g["%s%d" % (pre, i)] for i in range(3)], g["targets"], anchor_vecs("yolov3")
    gamma = {"g15": 1.5, "g05": 0.5}.get(case, 1.5)
    p = [torch.from_numpy(x).clone().requires_grad_(True) for x in preds]
    loss, items = focal_oracle.compute_loss(p, torch.from_numpy(t), av, _hyp(80, gamma), 80, 1.0)
    loss.backward()
    np.testing.assert_allclose(items.numpy(), g["items_" + case], rtol=1e-5)
    for i, pi in enumerate(p):
        np.testing.assert_allclose(pi.grad.numpy(), g["dp%d_%s" % (i, case)], rtol=1e-5, atol=1e-7)


def test_oracle_focal_loss_changes_the_loss():
    """the fixture's focal terms differ from plain BCE, and the box term does not depend on gamma"""
    g = golden("focal_case")
    p = [torch.from_numpy(g["p%d" % i]) for i in range(3)]
    _, plain = orc.compute_loss(p, torch.from_numpy(g["targets"]), anchor_vecs("yolov3"), _hyp(80), 80, 1.0)
    assert plain[0] == pytest.approx(float(g["items_g15"][0]), rel=1e-6)
    assert abs(float(plain[1]) - float(g["items_g15"][1])) > 1.0 and abs(float(plain[2]) - float(g["items_g15"][2])) > 1.0


@pytest.mark.parametrize("name", ["yolov2-tiny", "yolov3-tiny-nc100"])
def test_oracle_reproduces_wide_head_training_losses(name):
    import models
    g = golden("%s_128_train" % name)
    path, nc = (cfg_path(name), 80) if name == "yolov2-tiny" else (nc100_cfg(), 100)
    from utils.parse_config import parse_model_cfg
    defs = parse_model_cfg(path)[1:]
    sd = orc.synth_state_dict(models.Darknet(path).state_dict(), 0)
    x = orc.synth_images(4, 128, 128, seed=0)
    t = orc.synth_targets(4, 6, nc, seed=1)
    with torch.no_grad():
        p, _ = orc.darknet_forward(defs, sd, x, name, training=True)
    for i, pi in enumerate(p):
        np.testing.assert_allclose(pi.numpy(), g["p%d" % i], rtol=1e-3, atol=1e-3)
    _, items = orc.compute_loss([torch.from_numpy(g["p%d" % i]) for i in range(len(p))], t,
                                _anchor_vecs_of(path, name), _hyp(nc), nc, 1.0)
    np.testing.assert_allclose(items.numpy(), g["items"], rtol=1e-5)


def _train_plan(path, S=64):
    import models
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainPlan, TrainShared
    dev = torch.device("cpu")
    m = models.Darknet(path)
    return TrainPlan(m, (2, 3, S, S), dev, False, SlotStore(dev), TrainShared(dev))


def _heads(plan):
    return [r for r in plan.convs if r.head]


@pytest.mark.parametrize("name,cout,width", [("yolov2", 425, 432), ("yolov2-tiny", 425, 432),
                                             ("yolov3-tiny-nc100", 315, 320)])
def test_training_plan_builds_wide_heads(name, cout, width):
    plan = _train_plan(nc100_cfg() if name == "yolov3-tiny-nc100" else cfg_path(name))
    heads = _heads(plan)
    assert heads and all(r.Cout == cout and r.Cpad == width for r in heads)
    for r in heads:
        assert r.y.buf.shape[-1] == width and r.y.buf.dtype == torch.float32
        g = plan.grad_of[id(r.y)]
        assert g.C == width and tuple(g.buf.shape[1:]) == (r.y.H, r.y.W, width)
        assert tuple(r.w16.shape) == (width, 1, 1, r.Ipad)


@pytest.mark.parametrize("name", ["yolov3", "yolov3-tiny", "yolov4", "yolov3-mobilenet", "yolov3-tiny-nc1"])
def test_training_plan_keeps_256_wide_stock_heads(name):
    """255-filter heads (80 classes) and 18-filter heads (1 class) keep the 256-wide layout they always had"""
    from b200yolo import cfggen
    if name == "yolov3-tiny-nc1":
        path = os.path.join(tempfile.mkdtemp(prefix="b2y_nc1_"), name + ".cfg")
        with open(path, "w") as f:
            f.write(cfggen.cfg_text("yolov3-tiny", classes=1))
    else:
        path = cfg_path(name)
    plan = _train_plan(path)
    heads = _heads(plan)
    assert heads and all(r.Cpad == 256 for r in heads)
    for r in heads:
        assert r.Cout == (18 if name == "yolov3-tiny-nc1" else 255)
        assert r.y.buf.shape[-1] == 256
        assert plan.grad_of[id(r.y)].buf.shape[-1] == 256


def test_head_width():
    from b200yolo.train_engine import head_width
    assert [head_width(c) for c in (18, 255, 256, 257, 315, 425)] == [256, 256, 256, 272, 320, 432]
