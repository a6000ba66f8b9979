"""GPU: heads wider than 256 outputs (yolov2 / yolov2-tiny: 425, yolov3-tiny with 100 classes: 315) and the focal loss,
from the kernels up to training steps, against the fixtures the reference produced (oracle/gen_golden_heads.py) and the
oracle."""
import os
import tempfile

import numpy as np
import pytest
import torch

from helpers import anchor_vecs, attach_hyp, build_model, cfg_path, golden, orc
from oracle import focal_oracle
from test_gpu_kernels import conv_case
from test_gpu_train_kernels import conv_grads_case

pytestmark = pytest.mark.gpu

# the gates of tests/test_gpu_model.py (eval) and tests/test_gpu_train_model.py (training step)
BOX_REL_TOL_FP32REF, PROB_ABS_TOL_FP32REF = 3e-2, 1.5e-2
BOX_REL_TOL_EMU, PROB_ABS_TOL_EMU = 1e-2, 5e-3
POLICY_SLACK, P_ABS_FLOOR, LOSS_REL_FLOOR, NORM_REL_FLOOR, STAT_TOL = 2.0, 0.02, 5e-3, 0.02, 2e-2

_NC100 = []


def _nc100_path():
    from b200yolo import cfggen
    if not _NC100:
        path = os.path.join(tempfile.mkdtemp(prefix="b2y_nc100_"), "yolov3-tiny-nc100.cfg")
        with open(path, "w") as f:
            f.write(cfggen.cfg_text("yolov3-tiny", classes=100))
        _NC100.append(path)
    return _NC100[0]


def _model(name, device="cuda"):
    """(model with the synthetic weights of seed 0, cfg path, module defs, number of classes)"""
    import models
    from utils.parse_config import parse_model_cfg
    if name == "yolov3-tiny-nc100":
        path, nc = _nc100_path(), 100
    else:
        path, nc = cfg_path(name), 80
    m = models.Darknet(path)
    m.load_state_dict(orc.synth_state_dict(m.state_dict(), 0))
    return attach_hyp(m.to(device), nc), path, parse_model_cfg(path)[1:], nc


def _anchor_vecs(defs, name):
    ys = [d for d in defs if d['type'] == 'yolo']
    return [torch.as_tensor(np.asarray(d['anchors'])[d['mask']], dtype=torch.float32) / s
            for d, s in zip(ys, orc.yolo_strides(name, len(ys)))]


# ---- kernels on the head shapes ---------------------------------------------------------------------------------------
HEAD_CONV_CASES = [
    (2, 13, 13, 1024, 425, 1, 1, "linear", False, True, 0, 0),    # yolov2 head, fp32 out, clipped last N tile
    (2, 13, 13, 1024, 432, 1, 1, "linear", False, True, 0, 0),    # the same run at its padded width
    (2, 8, 8, 512, 320, 1, 1, "linear", False, True, 0, 0),       # 3 * (5 + 100) = 315 padded to 320
]


@pytest.mark.parametrize("case", HEAD_CONV_CASES, ids=[str(c) for c in HEAD_CONV_CASES])
def test_wide_head_conv_forward(case):
    err, rms = conv_case(*case)
    assert err <= 2e-5 * max(rms, 1.0), "max err %g rms %g" % (err, rms)


HEAD_GRAD_CASES = [
    (2, 13, 13, 1024, 432, 1, 1),   # data gradient K = 432, weight gradient over 432 output channels
    (2, 8, 8, 512, 320, 1, 1),      # K = 320
    (2, 16, 16, 256, 320, 1, 1),    # 320 output channels, split-K weight gradient
]


@pytest.mark.parametrize("case", HEAD_GRAD_CASES, ids=[str(c) for c in HEAD_GRAD_CASES])
def test_wide_head_conv_gradients(case):
    e_dx, e_dw = conv_grads_case(*case)
    print("\n%s dx err/rms=%.3g dw err/rms=%.3g" % (case, e_dx, e_dw))
    assert e_dx < 6e-3 and e_dw < 2e-4


# ---- focal loss -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["g15", "g05", "sat", "dup"])
def test_focal_loss_parity_fp32(case):
    """compute_loss with hyp['fl_gamma'] > 0 on the reference's focal_case: items and d loss / d p at rel 1e-4.
    'sat' sets every objectness / class logit to +-30 (gamma 1.5), 'dup' puts several targets in one cell."""
    from utils import utils as my_utils
    g = golden("focal_case")
    if case == "dup":
        model = attach_hyp(build_model("yolov3-tiny", device="cuda"))
        preds, t = [g["dup_p0"], g["dup_p1"]], g["dup_targets"]
    else:
        model = attach_hyp(build_model("yolov3", device="cuda"))
        pre = "sat_p" if case == "sat" else "p"
        preds, t = [g["%s%d" % (pre, i)] for i in range(3)], g["targets"]
    model.hyp['fl_gamma'] = {"g15": 1.5, "g05": 0.5}.get(case, 1.5)
    p = [torch.from_numpy(x).cuda().requires_grad_(True) for x in preds]
    loss, items = my_utils.compute_loss(p, torch.from_numpy(t).cuda(), model)
    loss.backward()
    np.testing.assert_allclose(items.cpu().numpy(), g["items_" + case], rtol=1e-4)
    for i, pi in enumerate(p):
        assert torch.isfinite(pi.grad).all()
        np.testing.assert_allclose(pi.grad.cpu().numpy(), g["dp%d_%s" % (i, case)], rtol=1e-4, atol=1e-6)


def test_focal_loss_training_step():
    """a yolov3-tiny training step with fl_gamma 1.5 through the engine: loss items against the fp32 oracle, as close as
    the fp16 precision policy lets the oracle itself get"""
    from utils import utils as my_utils
    model, path, defs, nc = _model("yolov3-tiny")
    model.train()
    model.hyp['fl_gamma'] = 1.5
    x = orc.synth_images(4, 128, 128, seed=0)
    t = orc.synth_targets(4, 6, 80, seed=1)
    pred, _ = model(x.cuda())
    loss, items = my_utils.compute_loss(pred, t.cuda(), model)
    loss.backward()
    torch.cuda.synchronize()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())
    sd = orc.synth_state_dict(model.state_dict(), 0)
    av, hyp = anchor_vecs("yolov3-tiny"), dict(model.hyp)
    with torch.no_grad():
        p32, _ = orc.darknet_forward(defs, sd, x, "yolov3-tiny", training=True)
        p16, _ = orc.darknet_forward(defs, sd, x, "yolov3-tiny", training=True, emulate_fp16=True)
    _, ref = focal_oracle.compute_loss(p32, t, av, hyp, 80, 1.0)
    _, yard = focal_oracle.compute_loss(p16, t, av, hyp, 80, 1.0)
    _, plain = orc.compute_loss(p32, t, av, dict(hyp, fl_gamma=0.0), 80, 1.0)
    rel = lambda a: float(((a - ref).abs() / ref.abs()).max())
    mine = items.cpu()
    print("\n[focal training step] engine %s | oracle fp32 %s | items rel engine %.3g / policy yardstick %.3g"
          % (mine.tolist(), ref.tolist(), rel(mine), rel(yard)))
    assert rel(mine) <= POLICY_SLACK * rel(yard) + LOSS_REL_FLOOR
    assert rel(plain) > 0.1          # the focal terms are really in the step


# ---- wide heads through the engine ------------------------------------------------------------------------------------
def _eval_errs(got, ref):
    box_rel = ((got[..., :4] - ref[..., :4]).abs() / ref[..., :4].abs().clamp(min=1.0)).max().item()
    prob = (got[..., 4:] - ref[..., 4:]).abs().max().item()
    return box_rel, prob


def test_yolov2_tiny_eval_parity():
    """one 425-wide head: fp32 and uint8 input against the reference's fp32 output and the fp16-policy oracle"""
    g = golden("yolov2-tiny_96_eval")
    model, path, defs, nc = _model("yolov2-tiny")
    model.eval()
    x = orc.synth_images(2, 96, 96, seed=3)
    u8 = torch.round(x * 256.0).to(torch.uint8)
    with torch.no_grad():
        io, p, _ = model(x.cuda())
        io_u8, p_u8, _ = model(u8.cuda())
    torch.cuda.synchronize()
    assert io.shape == g["io"].shape and len(p) == 1 and p[0].shape[-1] == 85 and p[0].shape[1] == 5
    assert torch.equal(io, io_u8) and torch.equal(p[0], p_u8[0])
    sd = orc.synth_state_dict(model.state_dict(), 0)
    with torch.no_grad():
        io_emu, _ = orc.darknet_forward(defs, sd, x, "yolov2-tiny", emulate_fp16=True)
    be, pe = _eval_errs(io.cpu(), io_emu)
    bf, pf = _eval_errs(io.cpu(), torch.from_numpy(g["io"]))
    print("\n[yolov2-tiny 96x96] vs fp16-policy oracle: box_rel=%.3g prob_abs=%.3g | vs fp32 reference: box_rel=%.3g "
          "prob_abs=%.3g" % (be, pe, bf, pf))
    assert be <= BOX_REL_TOL_EMU and pe <= PROB_ABS_TOL_EMU
    assert bf <= BOX_REL_TOL_FP32REF and pf <= PROB_ABS_TOL_FP32REF


@pytest.mark.parametrize("name", ["yolov2-tiny", "yolov3-tiny-nc100"])
def test_wide_head_train_step_parity(name):
    """test_train_step_parity's gates on the wide-head fixtures"""
    from utils import utils as my_utils
    g = golden("%s_128_train" % name)
    model, path, defs, nc = _model(name)
    model.train()
    x = orc.synth_images(4, 128, 128, seed=0).cuda()
    t = orc.synth_targets(4, 6, nc, seed=1).cuda()
    pred, feats = model(x)
    loss, items = my_utils.compute_loss(pred, t, model)
    loss.backward()
    torch.cuda.synchronize()
    names = [str(n) for n in g["grad_names"]]
    ref_norm = dict(zip(names, g["grad_norms"]))
    params = dict(model.named_parameters())
    for k in names:
        assert params[k].grad is not None and torch.isfinite(params[k].grad).all(), "bad gradient for %s" % k
    import models
    sd = orc.synth_state_dict(models.Darknet(path).state_dict(), 0)
    for k, v in sd.items():
        if v.dtype.is_floating_point and not k.endswith(('running_mean', 'running_var')):
            v.requires_grad_(True)
    pe, _ = orc.darknet_forward(defs, sd, x.cpu(), name, training=True, emulate_fp16=True)
    le, ie = orc.compute_loss(pe, t.cpu(), _anchor_vecs(defs, name), dict(model.hyp), nc, 1.0)
    le.backward()

    def dev_p(ps):
        return max((pi.detach().cpu() - torch.from_numpy(g["p%d" % i])).abs().max().item() for i, pi in enumerate(ps))

    def dev_items(it):
        return float((np.abs(it.detach().cpu().numpy() - g["items"]) / np.abs(g["items"])).max())

    def dev_norms(get):
        return np.array([abs(get(k) - ref_norm[k]) / (ref_norm[k] + 1e-8) for k in names])

    yard_p, mine_p = dev_p(pe), dev_p(pred)
    yard_l, mine_l = dev_items(ie), dev_items(items)
    yard_n = dev_norms(lambda k: float(sd[k].grad.norm()))
    mine_n = dev_norms(lambda k: float(params[k].grad.norm()))
    stat_err = 0.0
    msd = model.state_dict()
    for k in g.files:
        if k.startswith("stat::"):
            stat_err = max(stat_err, float((msd[k[6:]].cpu() - torch.from_numpy(g[k])).abs().max()))
    print("\n[%s train vs fp32 reference] engine / policy-yardstick: max|dp| %.3g / %.3g | loss items rel %.3g / %.3g | "
          "grad-norm rel median %.3g / %.3g  worst %.3g / %.3g | running-stat abs %.3g"
          % (name, mine_p, yard_p, mine_l, yard_l, np.median(mine_n), np.median(yard_n), mine_n.max(), yard_n.max(),
             stat_err))
    assert mine_p <= POLICY_SLACK * yard_p + P_ABS_FLOOR
    assert mine_l <= POLICY_SLACK * yard_l + LOSS_REL_FLOOR
    assert np.median(mine_n) <= POLICY_SLACK * np.median(yard_n) + NORM_REL_FLOOR
    assert mine_n.max() <= POLICY_SLACK * yard_n.max() + 5 * NORM_REL_FLOOR
    assert stat_err < STAT_TOL
    for k in names[-4:]:                      # the head conv and the BatchNorm before it, element-wise
        ref = torch.from_numpy(g["grad::" + k]).float()      # (fp16 for the 435k-weight yolov2-tiny head)
        err = ((params[k].grad.cpu() - ref).abs().max() / ref.abs().max().clamp(min=1e-12)).item()
        yard = ((sd[k].grad - ref).abs().max() / ref.abs().max().clamp(min=1e-12)).item()
        assert err <= POLICY_SLACK * yard + 0.02, (k, err, yard)
    assert len(feats) > 0


def test_yolov2_tiny_graph_replay_matches_eager_training():
    """test_graph_replay_matches_eager_training on the 425-wide head"""
    from utils import utils as my_utils
    x = orc.synth_images(4, 128, 128, seed=0).cuda()
    t = orc.synth_targets(4, 6, 80, seed=1).cuda()
    res = {}
    for graphed in (False, True):
        model = _model("yolov2-tiny")[0].train()
        model.use_cuda_graph = graphed
        losses, grads = [], []
        for _ in range(4):                       # eager, capture, replay, replay
            model.zero_grad(set_to_none=True)
            pred, _ = model(x)
            loss, _ = my_utils.compute_loss(pred, t, model)
            loss.backward()
            losses.append(float(loss.detach()))
            grads.append({k: p.grad.detach().clone() for k, p in model.named_parameters()})
        res[graphed] = (losses, grads)
    le, lg = res[False][0], res[True][0]
    print("\n[yolov2-tiny] eager losses %s\n      graph losses %s" % (le, lg))
    assert all(np.isfinite(lg))
    assert max(abs(a - b) / abs(a) for a, b in zip(le, lg)) < 2e-3
    assert max(abs(a - lg[0]) / abs(lg[0]) for a in lg) < 2e-3

    def worst(ga, gb):
        return max(float((ga[k] - gb[k]).norm() / (ga[k].norm() + 1e-12)) for k in ga)
    noise = worst(res[False][1][0], res[False][1][3])
    replay = worst(res[True][1][0], res[True][1][3])
    cross = worst(res[False][1][3], res[True][1][3])
    print("      eager-vs-eager %.3g  eager-vs-replay %.3g  model-vs-model %.3g" % (noise, replay, cross))
    assert replay < max(5e-2, 3 * noise)
    assert cross < max(5e-2, 3 * noise)


def test_nc100_flat_sink_matches_plain_autograd():
    """test_flat_sink_matches_plain_autograd on the 100-class yolov3-tiny (two 315-wide heads)"""
    from utils import utils as my_utils
    from b200yolo.parallel import FlatDataParallel
    B, S = 8, 416
    x = orc.synth_images(B, S, S, seed=10).cuda()
    t = orc.synth_targets(B, 6, 100, seed=20).cuda()
    plain = _model("yolov3-tiny-nc100")[0].train()
    plain.use_cuda_graph = False
    runs = []
    for _ in range(2):
        plain.zero_grad(set_to_none=True)
        pred, _ = plain(x)
        loss, _ = my_utils.compute_loss(pred, t, plain)
        loss.backward()
        runs.append({k: p.grad.detach().clone() for k, p in plain.named_parameters()})
    wrapped = _model("yolov3-tiny-nc100")[0].train()
    dp = FlatDataParallel(wrapped)
    dp.zero_grad()
    pred, _ = dp(x)
    loss2, _ = my_utils.compute_loss(pred, t, dp)
    loss2.backward()
    torch.cuda.synchronize()
    noise = max(float((runs[0][k] - runs[1][k]).norm() / (runs[0][k].norm() + 1e-12)) for k in runs[0])
    errs = sorted(((float((dp.grad_views[id(p)] - runs[0][n]).norm() / (runs[0][n].norm() + 1e-12)), n)
                   for n, p in zip(dp.names, dp.params)), reverse=True)
    print("\n[nc100 sink vs plain] loss %.6f vs %.6f | run-to-run noise %.3g | worst sink-vs-plain %s"
          % (float(loss2), float(loss), noise, errs[:3]))
    assert abs(float(loss2) - float(loss)) / abs(float(loss)) < 1e-3
    assert errs[0][0] < max(1e-3, 3 * noise)
