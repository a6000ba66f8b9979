"""GPU: google QAT (quantized=1) of yolov3-mobilenet.  Its [depthwise] blocks (Conv2d(groups=C) + batch-statistics
BatchNorm2d + activation) and [se] layers stay in float, as in the reference, and run on the fp32 NHWC kernels of
depthwise.cu / bn_train.cu through b200yolo/qat.py.  Kernels against float64 torch; the full training step and the eval
forward against the reference's own run (oracle/gen_golden_qat_mobilenet.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import attach_hyp, cfg_path, golden, orc

pytestmark = pytest.mark.gpu

STEPS = 100


def _model():
    import models
    sd = orc.synth_state_dict(models.Darknet(cfg_path("yolov3-mobilenet")).state_dict(), 0)
    qm = models.Darknet(cfg_path("yolov3-mobilenet"), quantized=1, a_bit=8, w_bit=8, shortcut_way=1, steps=STEPS)
    new = {}
    for k, v in qm.state_dict().items():      # as oracle/gen_golden_qat_mobilenet.py loads the reference's model
        i = k.split('.')[1]
        if k.endswith('Conv2d.weight'):
            new[k] = sd[k]
        elif k.endswith('Conv2d.gamma'):
            new[k] = sd.get('module_list.%s.BatchNorm2d.weight' % i, torch.ones_like(v))
        elif k.endswith('Conv2d.beta'):
            new[k] = sd.get('module_list.%s.BatchNorm2d.bias' % i, torch.zeros_like(v))
        elif k.endswith('Conv2d.bias') and ('module_list.%s.Conv2d.bias' % i) in sd:
            new[k] = sd['module_list.%s.Conv2d.bias' % i]
        elif ('.DepthWise2d.' in k or '.BatchNorm2d.' in k or '.se.' in k) and k in sd:
            new[k] = sd[k]
        else:
            new[k] = v
    qm.load_state_dict(new)
    return attach_hyp(qm.cuda())


def _act64(z, act):
    if act == 'relu6':
        return z.clamp(0, 6)
    if act == 'h_swish':
        return z * (z + 3).clamp(0, 6) / 6
    if act == 'relu':
        return z.clamp(min=0)
    return z


def _rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp(min=1e-30))


@pytest.mark.parametrize("C,k,s,act", [(16, 3, 1, 'relu'), (24, 3, 1, 'relu6'), (40, 5, 2, 'relu6'),
                                       (72, 5, 2, 'h_swish'), (120, 5, 1, 'h_swish'), (184, 3, 1, 'h_swish'),
                                       (200, 3, 2, 'h_swish'), (960, 5, 1, 'linear')])
@pytest.mark.parametrize("training", [True, False])
def test_depthwise_block_matches_torch(C, k, s, act, training):
    from b200yolo import qat
    g = torch.Generator().manual_seed(C * 10 + k + s)
    x = torch.randn(2, 13, 11, C, generator=g).cuda()
    w = (torch.randn(C, 1, k, k, generator=g) / k).cuda()
    gamma, beta = (torch.rand(C, generator=g) + 0.5).cuda(), (0.1 * torch.randn(C, generator=g)).cuda()
    rm, rv = (0.1 * torch.randn(C, generator=g)).cuda(), (torch.rand(C, generator=g) + 0.5).cuda()
    gy = torch.randn(2, (13 + 2 * (k // 2) - k) // s + 1, (11 + 2 * (k // 2) - k) // s + 1, C, generator=g).cuda()
    # ours
    xs, ws, gs, bs = [t.clone().requires_grad_(True) for t in (x, w, gamma, beta)]
    rm1, rv1 = rm.clone(), rv.clone()
    y = qat.DepthwiseBlockFn.apply(xs, ws, gs, bs, rm1, rv1, k, s, k // 2, act, 0.1, training, 0.1, 1e-5)
    y.backward(gy)
    # float64 torch
    xr, wr, gr, br = [t.double().clone().requires_grad_(True) for t in (x, w, gamma, beta)]
    rm2, rv2 = rm.double().clone(), rv.double().clone()
    z = F.conv2d(xr.permute(0, 3, 1, 2), wr, None, s, k // 2, 1, C)
    yr = _act64(F.batch_norm(z, rm2, rv2, gr, br, training, 0.1, 1e-5), act).permute(0, 2, 3, 1)
    yr.backward(gy.double())
    errs = dict(y=_rel(y, yr), dx=_rel(xs.grad, xr.grad), dw=_rel(ws.grad, wr.grad), dgamma=_rel(gs.grad, gr.grad),
                dbeta=_rel(bs.grad, br.grad), rm=_rel(rm1, rm2), rv=_rel(rv1, rv2))
    print("\n[depthwise C=%d k=%d s=%d %s %s] %s" % (C, k, s, act, "train" if training else "eval",
                                                    " ".join("%s=%.2g" % kv for kv in errs.items())))
    assert max(errs.values()) < 2e-5, errs


@pytest.mark.parametrize("C,hw", [(72, (7, 9)), (120, (13, 13)), (480, (4, 4)), (672, (3, 5)), (960, (2, 2))])
def test_se_matches_torch(C, hw):
    from b200yolo import qat
    g = torch.Generator().manual_seed(C)
    Cr = C // 4
    x = torch.randn(3, hw[0], hw[1], C, generator=g).cuda()
    w1 = (torch.randn(Cr, C, generator=g) / C ** 0.5).cuda()
    w2 = (torch.randn(C, Cr, generator=g) * 3 / Cr ** 0.5).cuda()   # gates on both sides of the hard-sigmoid's knees
    gy = torch.randn_like(x)
    xs, a, b = [t.clone().requires_grad_(True) for t in (x, w1, w2)]
    y = qat.SEFn.apply(xs, a, b)
    y.backward(gy)
    xr, ar, br = [t.double().clone().requires_grad_(True) for t in (x, w1, w2)]
    gate = F.relu6(F.linear(F.relu(F.linear(xr.mean((1, 2)), ar)), br) + 3) / 6
    yr = xr * gate[:, None, None, :]
    yr.backward(gy.double())
    errs = dict(y=_rel(y, yr), dx=_rel(xs.grad, xr.grad), dw1=_rel(a.grad, ar.grad), dw2=_rel(b.grad, br.grad))
    print("\n[se C=%d hw=%s] %s" % (C, hw, " ".join("%s=%.2g" % kv for kv in errs.items())))
    assert max(errs.values()) < 2e-5, errs


@pytest.mark.parametrize("I,O", [(16, 24), (24, 72), (40, 120), (72, 40), (120, 184), (184, 200), (200, 80)])
def test_qat_conv_pads_odd_widths(I, O):
    """ConvFn pads K and Cout to the MMA granule of 16: output, dx and dw against float64 torch at MobileNet widths"""
    from b200yolo import qat
    g = torch.Generator().manual_seed(I * 1000 + O)
    # inputs and weights on the fp16 grid, as the fake-quantised tensors of the QAT graph are
    x = torch.randn(2, 9, 9, I, generator=g).half().float().cuda()
    w = (torch.randn(O, I, 1, 1, generator=g) / I ** 0.5).half().float().cuda()
    gy = torch.randn(2, 9, 9, O, generator=g).cuda()
    xs, ws = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = qat.conv2d(xs, ws, 1, 1, 0)
    y.backward(gy)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = F.conv2d(xr.permute(0, 3, 1, 2), wr).permute(0, 2, 3, 1)
    yr.backward(gy.double())
    errs = dict(y=_rel(y, yr), dx=_rel(xs.grad, xr.grad), dw=_rel(ws.grad, wr.grad))
    print("\n[qat conv %d->%d] %s" % (I, O, " ".join("%s=%.2g" % kv for kv in errs.items())))
    assert errs["y"] < 1e-6 and errs["dx"] < 5e-3 and errs["dw"] < 2e-3, errs


def _step(qm):
    from utils import utils as my_utils
    x = orc.synth_images(2, 64, 64, seed=0).cuda()
    t = orc.synth_targets(2, 6, 80, seed=1).cuda()
    pred, _ = qm(x)
    loss, items = my_utils.compute_loss(pred, t, qm)
    loss.backward()
    torch.cuda.synchronize()
    return pred, items


def test_mobilenet_qat_training_step_and_eval_match_reference():
    """the gates of tests/test_gpu_qat.py (yolov3 / yolov3-tiny QAT) on the 107-layer MobileNet QAT graph"""
    g = golden("yolov3-mobilenet_64_qat1")
    qm = _model().train()
    pred, items = _step(qm)
    items_rel = float((np.abs(items.detach().cpu().numpy() - g["items"]) / np.abs(g["items"])).max())
    params = dict(qm.named_parameters())
    names = [str(n) for n in g["grad_names"]]
    ref = dict(zip(names, g["grad_norms"]))
    missing = [k for k in names if params[k].grad is None]
    floor = 1e-3 * float(np.median(list(ref.values())))
    rel = {k: abs(float(params[k].grad.norm()) - v) / max(v, floor) for k, v in ref.items() if params[k].grad is not None}
    dw_rel = [v for k, v in rel.items() if '.DepthWise2d.' in k or '.BatchNorm2d.' in k]
    se_rel = [v for k, v in rel.items() if '.se.' in k]
    sd = qm.state_dict()
    sn, sv = [str(n) for n in g["scale_names"]], g["scale_values"]
    diff = [k for k, v in zip(sn, sv) if abs(float(sd[k].reshape(-1)[0]) - float(v)) > 1e-6 * abs(float(v))]
    # the first depthwise block sits behind two QAT convs only: its running statistics and step counter are exact to fp32
    i0 = next(i for i, d in enumerate(qm.module_defs) if d['type'] == 'depthwise')
    first = {n: float((sd['module_list.%d.BatchNorm2d.%s' % (i0, n)].cpu() -
                       torch.from_numpy(g['state::module_list.%d.BatchNorm2d.%s' % (i0, n)])).abs().max())
             for n in ('running_mean', 'running_var')}
    nbt = [k for k in g.files if k.startswith('state::') and k.endswith('num_batches_tracked')]
    assert nbt and all(int(sd[k[7:]]) == int(g[k]) for k in nbt)
    print("\n[yolov3-mobilenet qat1 train step vs reference] loss items rel %.3g | grad-norm rel median %.3g worst %.3g "
          "(depthwise/BN median %.3g, SE median %.3g, %d params without grad) | scales differing %d of %d | first "
          "depthwise running stats abs %s" % (items_rel, np.median(list(rel.values())), max(rel.values()),
                                              np.median(dw_rel), np.median(se_rel), len(missing), len(diff), len(sn), first))
    qm.eval()
    with torch.no_grad():
        io, p, _ = qm(orc.synth_images(2, 64, 64, seed=5).cuda())
    ref_io = torch.from_numpy(g["eval_io"])
    close = float(torch.isclose(io.cpu(), ref_io, rtol=2e-2, atol=2e-2).float().mean())
    print("[yolov3-mobilenet qat1 eval after the step] fraction of io within 2e-2: %.4f" % close)
    assert not missing
    assert items_rel < 0.1
    assert np.median(list(rel.values())) < 0.5
    assert len(diff) <= 0.12 * len(sn)
    assert max(first.values()) < 1e-4
    assert torch.isfinite(io).all()


def test_mobilenet_qat_step_is_deterministic():
    grads = []
    for _ in range(2):
        qm = _model().train()
        _step(qm)
        grads.append({k: p.grad.detach().clone() for k, p in qm.named_parameters() if p.grad is not None})
    assert grads[0].keys() == grads[1].keys()
    bad = [k for k in grads[0] if not torch.equal(grads[0][k], grads[1][k])]
    assert not bad, bad[:5]


def test_mobilenet_qat_flat_sgd_step():
    """FlatDataParallel + FlatSGD over train.py's quantized=1 parameter groups on the QAT MobileNet"""
    from b200yolo.optim import FlatSGD, train_param_groups
    from b200yolo.parallel import FlatDataParallel
    dp = FlatDataParallel(_model().train())
    pg0, pg1, pg2, _ = train_param_groups(dp, 1)
    opt = FlatSGD(dp, pg0, lr=0.01, momentum=0.9, nesterov=True)
    opt.add_param_group({'params': pg1, 'weight_decay': 5e-4})
    opt.add_param_group({'params': pg2})
    before = dp.flat_param.clone()
    from utils import utils as my_utils
    pred, _ = dp(orc.synth_images(2, 64, 64, seed=0).cuda())
    loss, _ = my_utils.compute_loss(pred, orc.synth_targets(2, 6, 80, seed=1).cuda(), dp.module)
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    moved = dp.flat_param - before
    assert torch.isfinite(dp.flat_param).all()
    assert float(moved.abs().max()) > 0
    i0 = next(i for i, d in enumerate(dp.module.module_defs) if d['type'] == 'depthwise')
    w = dp.module.module_list[i0][0].weight
    assert w.grad is not None and float(w.grad.abs().max()) > 0
