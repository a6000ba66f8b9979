"""GPU: training step parity (forward with batch-stat BN, YOLO loss, full backward) of the H100 engine against the
fixtures produced by the reference itself on CPU fp32 (tests/golden/*_64_train.npz)."""
import numpy as np
import pytest
import torch

from helpers import anchor_vecs, attach_hyp, build_model, cfg_path, golden, module_defs, orc

pytestmark = pytest.mark.gpu

# A deep, randomly initialised Darknet in train mode (batch-statistics BN over as few as 64 samples) amplifies 16-bit
# rounding chaotically: the ORACLE itself moves by max|dp| = 0.018 (tiny) / 0.12 (yolov3) / 1.3 (yolov4) between fp32 and
# the fp16 activation policy.  The gate is therefore relative to that yardstick: the engine must be as close to the
# reference's fp32 result as the precision policy permits (factor POLICY_SLACK), plus small absolute floors.  Kernel
# correctness proper is gated per kernel on identical inputs in tests/test_gpu_train_kernels.py.
POLICY_SLACK = 2.0
P_ABS_FLOOR = 0.02
LOSS_REL_FLOOR = 5e-3
NORM_REL_FLOOR = 0.02
STAT_TOL = 2e-2


@pytest.mark.parametrize("name", ["yolov3-tiny", "yolov3", "yolov4"])
def test_train_step_parity(name):
    from utils import utils as my_utils
    import models as _models
    g = golden("%s_128_train" % name)                       # the reference itself, fp32 CPU
    model = attach_hyp(build_model(name, device="cuda")).train()
    x = orc.synth_images(4, 128, 128, seed=0).cuda()
    t = orc.synth_targets(4, 6, 80, seed=1).cuda()
    pred, feats = model(x)
    loss, items = my_utils.compute_loss(pred, t, model)
    loss.backward()
    torch.cuda.synchronize()
    names = [str(n) for n in g["grad_names"]]
    ref_norm = dict(zip(names, g["grad_norms"]))
    params = dict(model.named_parameters())
    for k in names:
        assert params[k].grad is not None and torch.isfinite(params[k].grad).all(), "bad gradient for %s" % k

    # yardstick: the oracle under the engine's forward precision policy (fp16 weights / activations, fp32 backward)
    sd = orc.synth_state_dict(_models.Darknet(cfg_path(name)).state_dict(), 0)
    for k, v in sd.items():
        if v.dtype.is_floating_point and not k.endswith(('running_mean', 'running_var')):
            v.requires_grad_(True)
    pe, _ = orc.darknet_forward(module_defs(name), sd, x.cpu(), name, training=True, emulate_fp16=True)
    le, ie = orc.compute_loss(pe, t.cpu(), anchor_vecs(name), dict(orc.DEFAULT_HYP), 80, 1.0)
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
    # last layers (head conv and the BN before it) see almost no accumulated rounding: element-wise check
    for k in names[-4:]:
        ref = torch.from_numpy(g["grad::" + k])
        err = ((params[k].grad.cpu() - ref).abs().max() / ref.abs().max().clamp(min=1e-12)).item()
        yard = ((sd[k].grad - ref).abs().max() / ref.abs().max().clamp(min=1e-12)).item()
        assert err <= POLICY_SLACK * yard + 0.02, (k, err, yard)
    assert len(feats) > 0


def test_train_step_then_optimizer_changes_output():
    """weights change -> the plan re-packs them; two steps with torch SGD decrease the loss on a fixed batch."""
    from utils import utils as my_utils
    model = attach_hyp(build_model("yolov3-tiny", device="cuda")).train()
    opt = torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, nesterov=True)
    x = orc.synth_images(4, 128, 128, seed=0).cuda()
    t = orc.synth_targets(4, 6, 80, seed=1).cuda()
    losses = []
    for _ in range(4):
        opt.zero_grad()
        pred, _ = model(x)
        loss, _ = my_utils.compute_loss(pred, t, model)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


@pytest.mark.parametrize("name", ["yolov3-tiny", "yolov4"])
def test_graph_replay_matches_eager_training(name):
    """Steps 3+ replay the captured forward / backward CUDA graphs.  With frozen parameters every step computes the
    same thing, so the replayed loss and gradients must equal the eagerly launched ones up to the fp32 reordering of
    the atomics (split-K weight gradient, BN sums) -- no chaotic amplification across optimiser steps involved."""
    from utils import utils as my_utils
    x = orc.synth_images(4, 128, 128, seed=0).cuda()
    t = orc.synth_targets(4, 6, 80, seed=1).cuda()
    res = {}
    for graphed in (False, True):
        model = attach_hyp(build_model(name, device="cuda")).train()
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
    print("\n[%s] eager losses %s\n      graph losses %s" % (name, le, lg))
    assert all(np.isfinite(lg))
    ltol = 2e-3 if name == "yolov3-tiny" else 3e-2     # yolov4 at this size amplifies the atomics' fp32 reordering
    assert max(abs(a - b) / abs(a) for a, b in zip(le, lg)) < ltol
    assert max(abs(a - lg[0]) / abs(lg[0]) for a in lg) < ltol          # replays reproduce the eager step

    def worst(ga, gb):
        d = sorted(((float((ga[k] - gb[k]).norm() / (ga[k].norm() + 1e-12)), k, float(ga[k].norm())) for k in ga),
                   reverse=True)
        return d[:3]
    noise = worst(res[False][1][0], res[False][1][3])         # eager step 1 vs eager step 4: atomics reordering only
    replay = worst(res[True][1][0], res[True][1][3])          # same model: eager step 1 vs graph replay step 4
    cross = worst(res[False][1][3], res[True][1][3])
    print("      eager-vs-eager   ", noise, "\n      eager-vs-replay  ", replay, "\n      model-vs-model   ", cross)
    assert replay[0][0] < max(5e-2, 3 * noise[0][0])
    assert cross[0][0] < max(5e-2, 3 * noise[0][0])


@pytest.mark.parametrize("name,B,S", [("yolov3-tiny", 8, 416), ("yolov3", 8, 256)])
def test_flat_sink_matches_plain_autograd(name, B, S):
    """FlatDataParallel (world size 1): the training plan writes every gradient straight into the flat buffer (BatchNorm
    backward kernels, the table-driven weight-gradient unpack) -- the result must equal the plain autograd path (plan-owned
    buffers handed to .grad) up to the fp32 reordering of the split-K / BN-sum atomics."""
    from utils import utils as my_utils
    from b200yolo.parallel import FlatDataParallel
    x = orc.synth_images(B, S, S, seed=10).cuda()
    t = orc.synth_targets(B, 6, 80, seed=20).cuda()
    plain = attach_hyp(build_model(name, device="cuda")).train()
    plain.use_cuda_graph = False
    runs = []
    for _ in range(2):                       # twice: the run-to-run noise of the atomics is the yardstick
        plain.zero_grad(set_to_none=True)
        pred, _ = plain(x)
        loss, _ = my_utils.compute_loss(pred, t, plain)
        loss.backward()
        runs.append({k: p.grad.detach().clone() for k, p in plain.named_parameters()})
    wrapped = attach_hyp(build_model(name, device="cuda")).train()
    dp = FlatDataParallel(wrapped)
    dp.zero_grad()
    pred, _ = dp(x)
    loss2, _ = my_utils.compute_loss(pred, t, dp)
    loss2.backward()
    torch.cuda.synchronize()
    noise = max(float((runs[0][k] - runs[1][k]).norm() / (runs[0][k].norm() + 1e-12)) for k in runs[0])
    errs = sorted(((float((dp.grad_views[id(p)] - runs[0][n]).norm() / (runs[0][n].norm() + 1e-12)), n)
                   for n, p in zip(dp.names, dp.params)), reverse=True)
    print("\n[%s sink vs plain] loss %.6f vs %.6f | run-to-run noise %.3g | worst sink-vs-plain %s"
          % (name, float(loss2), float(loss), noise, errs[:3]))
    # (a randomly initialised batch-statistics network is chaotic in the backward direction: at 4x128x128 two runs of the
    #  SAME model differ by 9 % / 39 % element-wise in the early layers from the fp32 reordering of the atomics alone --
    #  measured -- so the comparison is made at sizes where every BatchNorm sees >= 512 samples, relative to that noise)
    assert abs(float(loss2) - float(loss)) / abs(float(loss)) < 1e-3
    assert errs[0][0] < max(1e-3, 3 * noise)
