"""GPU: TPSQ (quantized=2) of yolov3-mobilenet.  Every [depthwise] block is one quantised, BN-folded
TPSQ_BNFold_QuantizedConv2d_For_FPGA(groups=C): a statistics conv with the float weights and a conv with the folded,
power-of-two quantised weights, both on the fp32 NHWC kernels of depthwise.cu.  The kernels and one layer against
float64 torch (the layer against a float64 restatement of the reference module kept below); the layers on the
reference's own tensors, a full training step and the eval forward against the reference's own run
(oracle/gen_golden_qat2_mobilenet.py)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import attach_hyp, cfg_path, golden, orc

pytestmark = pytest.mark.gpu

STEPS = 100
# the shapes of test_gpu_qat_mobilenet.py::test_depthwise_block_matches_torch
SHAPES = [(16, 3, 1, 'relu'), (24, 3, 1, 'relu6'), (40, 5, 2, 'relu6'), (72, 5, 2, 'h_swish'), (120, 5, 1, 'h_swish'),
          (184, 3, 1, 'h_swish'), (200, 3, 2, 'h_swish'), (960, 5, 1, 'linear')]


def _model():
    import models
    sd = orc.synth_state_dict(models.Darknet(cfg_path("yolov3-mobilenet")).state_dict(), 0)
    qm = models.Darknet(cfg_path("yolov3-mobilenet"), quantized=2, a_bit=8, w_bit=8, shortcut_way=1, steps=STEPS)
    new = {}
    for k, v in qm.state_dict().items():      # as oracle/gen_golden_qat2_mobilenet.py loads the reference's model
        i = k.split('.')[1]
        if k.endswith(('Conv2d.weight', 'DepthWise2d.weight')):
            new[k] = sd[k]
        elif k.endswith(('Conv2d.gamma', 'DepthWise2d.gamma')):
            new[k] = sd.get('module_list.%s.BatchNorm2d.weight' % i, torch.ones_like(v))
        elif k.endswith(('Conv2d.beta', 'DepthWise2d.beta')):
            new[k] = sd.get('module_list.%s.BatchNorm2d.bias' % i, torch.zeros_like(v))
        elif k.endswith('Conv2d.bias') and ('module_list.%s.Conv2d.bias' % i) in sd:
            new[k] = sd['module_list.%s.Conv2d.bias' % i]
        elif '.se.' in k and k in sd:
            new[k] = sd[k]
        else:
            new[k] = v
    qm.load_state_dict(new)
    return attach_hyp(qm.cuda())


def _rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp(min=1e-30))


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _out_hw(k, s):
    return (13 + 2 * (k // 2) - k) // s + 1, (11 + 2 * (k // 2) - k) // s + 1


# ---- kernels ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,k,s,act", SHAPES)
def test_dwconv_stats_match_torch(C, k, s, act):
    from b200yolo import qat
    g = torch.Generator().manual_seed(C * 10 + k + s)
    x = torch.randn(2, 13, 11, C, generator=g)
    w = torch.randn(C, 1, k, k, generator=g) / k
    b = 0.1 * torch.randn(C, generator=g)
    # channel 0: |mean| ~ 1e3 from the input, std ~ 1; channel 1: the same from the bias
    x[..., 0] += 1000.0
    w[0] = 0.0
    w[0, 0, k // 2, k // 2] = 1.0
    b[1] = 1000.0
    mean, var = qat.dwconv_stats(x.cuda(), w.cuda(), b.cuda(), k, s, k // 2)
    z = F.conv2d(_nchw(x).double(), w.double(), b.double(), s, k // 2, 1, C)
    rm, rv = z.mean((0, 2, 3)), z.var((0, 2, 3))
    mean, var = mean.double().cpu(), var.double().cpu()
    e_mean = float(((mean - rm).abs() / (rm.abs() + rv.sqrt())).max())
    e_var = float(((var - rv).abs() / rv).max())
    print("\n[dwconv stats C=%d k=%d s=%d] mean %.2g var %.2g (channel 0 var %.6g ref %.6g)"
          % (C, k, s, e_mean, e_var, float(var[0]), float(rv[0])))
    assert e_mean < 1e-6 and e_var < 1e-6


@pytest.mark.parametrize("C,k,s,act", SHAPES)
def test_dwconv_stats_backward_matches_torch(C, k, s, act):
    """the statistics conv and the quantised conv on one input, W_q folded from the variance as in the layer: dx, dW_q
    and dw_s against float64 torch"""
    from b200yolo import qat
    g = torch.Generator().manual_seed(C * 10 + k + s + 1)
    p = k // 2
    x = torch.randn(2, 13, 11, C, generator=g)
    ws = torch.randn(C, 1, k, k, generator=g) / k
    wq0 = torch.randn(C, 1, k, k, generator=g) / k
    gamma = torch.rand(C, generator=g) + 0.5
    ho, wo = _out_hw(k, s)
    gq = torch.randn(2, ho, wo, C, generator=g)
    gm, gv = torch.randn(C, generator=g), torch.randn(C, generator=g)

    def run(x, ws, wq0, conv_stats, conv):
        mean, var = conv_stats(x, ws)
        wq = wq0 * (gamma.to(x) / torch.sqrt(var + 1e-5)).reshape(-1, 1, 1, 1)
        wq.retain_grad()
        y = conv(x, wq)
        ((y * gq.to(x)).sum() + (mean * gm.to(x)).sum() + (var * gv.to(x)).sum()).backward()
        return wq

    xs, wss, wqs = [t.cuda().requires_grad_(True) for t in (x, ws, wq0)]
    link = qat.DwGradLink()
    wq = run(xs, wss, wqs, lambda a, w: qat.dwconv_stats(a, w, None, k, s, p, link),
             lambda a, w: qat.dwconv2d(a, w, k, s, p, link))
    xr, wsr, wqr = [t.double().requires_grad_(True) for t in (x, ws, wq0)]

    def stats64(a, w):
        z = F.conv2d(_nchw(a), w, None, s, p, 1, C)
        return z.mean((0, 2, 3)), z.var((0, 2, 3))
    wq64 = run(xr, wsr, wqr, stats64, lambda a, w: F.conv2d(_nchw(a), w, None, s, p, 1, C).permute(0, 2, 3, 1))
    errs = dict(dx=_rel(xs.grad, xr.grad), dWq=_rel(wq.grad, wq64.grad), dws=_rel(wss.grad, wsr.grad),
                dwq0=_rel(wqs.grad, wqr.grad))
    print("\n[dwconv stats backward C=%d k=%d s=%d] %s" % (C, k, s, " ".join("%s=%.2g" % kv for kv in errs.items())))
    assert max(errs.values()) < 2e-5, errs


# ---- one layer against a float64 restatement of the reference module ------------------------------------------------
class _Pow2(torch.autograd.Function):
    """Search_Pow2 (reference quantized_TPSQ.py:29-63): nearest power of two, gradient scaled by output / input"""

    @staticmethod
    def forward(ctx, s):
        v = float(s)
        v = 2.0 ** -5 if v < 0 else min(v, 2.0 ** 13)
        ce, fl = 2.0 ** math.ceil(math.log2(v)), 2.0 ** math.floor(math.log2(v))
        P = ce if abs(ce - v) < abs(fl - v) else fl
        ctx.r = P / float(s)
        return torch.full_like(s, P)

    @staticmethod
    def backward(ctx, g):
        return g * ctx.r


class _Round(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return torch.sign(x) * torch.floor(x.abs() + 0.5)

    @staticmethod
    def backward(ctx, g):
        return g


def _tpsq64(x, scale, bits=8):
    """Quantizer.forward (reference :66-130): soft clamp, quantise, round, dequantise"""
    P = _Pow2.apply(scale)
    c = 0.5 * ((x + P).abs() - (x - P).abs())
    return _Round.apply(c * ((1 << (bits - 1)) - 1) / P) * P / (1 << (bits - 1))


def _act64(z, act):
    if act == 'relu6':
        return F.relu6(z)
    if act == 'h_swish':
        return z * F.relu6(z + 3.0) / 6.0
    if act == 'relu':
        return F.relu(z)
    return z


def _layer64(c, x, training, p):
    """TPSQ_BNFold_QuantizedConv2d_For_FPGA.forward (reference :404-589) for bn=1, bias=None, in float64 on a snapshot of
    the module's state; x NCHW.  Returns y and the leaves (weight, gamma, beta, weight scale, activation scale) and the
    running statistics after the call."""
    C, k, s = c.in_channels, c.kernel_size[0], c.stride[0]
    d = lambda t: t.detach().double().cpu().clone()  # noqa: E731
    w, gamma, beta = [d(t).requires_grad_(True) for t in (c.weight, c.gamma, c.beta)]
    ws, as_ = [d(q.scale).requires_grad_(True) for q in (c.weight_quantizer, c.activation_quantizer)]
    rm, rv, first_bn, step = d(c.running_mean), d(c.running_var), float(c.first_bn), float(c.step)
    bq = c.bias_quantizer
    if training:
        step += 1
        z = F.conv2d(x, w, None, s, p, 1, C)
        bm, bv = z.mean((0, 2, 3)), z.var((0, 2, 3))
        with torch.no_grad():
            if first_bn == 0 and not rm.any() and not rv.any():
                rm, rv = rm + bm, rv + bv
            else:
                rm, rv = rm * (1 - c.momentum) + bm * c.momentum, rv * (1 - c.momentum) + bv * c.momentum
        if step < c.freeze_step:
            sc = gamma / torch.sqrt(bv + c.eps)
            bias = beta - bm * sc
        else:
            sc = gamma / torch.sqrt(rv + c.eps)
            bias = beta - rm * sc
        # GlobalRangeTracker and Bias_Quantizer.update_params
        lo, hi = float(bias.detach().min()), float(bias.detach().max())
        if float(bq.range_tracker.first_w) != 0:
            lo, hi = min(lo, float(bq.range_tracker.min_val)), max(hi, float(bq.range_tracker.max_val))
        fmax = max(abs(lo), abs(hi))
        fl, ce = 2.0 ** math.floor(math.log2(fmax)), 2.0 ** math.ceil(math.log2(fmax))
        bscale = (ce if abs(ce - fmax) < abs(fl - fmax) else fl) / 128.0
    else:
        sc = gamma / torch.sqrt(rv + c.eps)
        bias = beta - rm * sc
        bscale = float(bq.scale)
    qw = _tpsq64(w * sc.reshape(-1, 1, 1, 1), ws)
    qb = torch.clamp(_Round.apply(bias / bscale), -128, 127) * bscale
    y = _tpsq64(_act64(F.conv2d(x, qw, qb, s, p, 1, C), c.activate), as_)
    return y, dict(weight=w, gamma=gamma, beta=beta, wscale=ws, ascale=as_), rm, rv


@pytest.mark.parametrize("C,k,s,act", [(72, 5, 2, 'relu6'), (120, 5, 1, 'h_swish'), (200, 3, 1, 'h_swish'),
                                       (960, 5, 1, 'relu6')])
@pytest.mark.parametrize("regime", ["first_step", "before_freeze", "after_freeze", "eval"])
def test_tpsq_depthwise_layer_matches_float64(C, k, s, act, regime):
    from utils.quantized.quantized_TPSQ import TPSQ_BNFold_QuantizedConv2d_For_FPGA
    g = torch.Generator().manual_seed(C + k + s)
    p = k // 2
    c = TPSQ_BNFold_QuantizedConv2d_For_FPGA(C, C, k, s, p, groups=C, bias=False, bn=1, activate=act, steps=STEPS).cuda()
    with torch.no_grad():
        c.weight.copy_(torch.randn(C, 1, k, k, generator=g) / k)
        c.gamma.copy_(torch.rand(C, generator=g) + 0.5)
        c.beta.copy_(0.1 * torch.randn(C, generator=g))
        c.activation_quantizer.warmup.zero_()                # a preset range: the warm-up search is not the subject
        c.activation_quantizer.scale.fill_(3.1)
        if regime != "first_step":
            c.running_mean.copy_(0.1 * torch.randn(C, generator=g))
            c.running_var.copy_(torch.rand(C, generator=g) + 0.5)
            c.first_bn.fill_(1)
            c.step.fill_({"before_freeze": 10, "after_freeze": c.freeze_step - 1, "eval": STEPS}[regime])
            c.bias_quantizer.scale.fill_(2.0 ** -6)
    training = regime != "eval"
    c.train(training)
    # the input on an activation grid, as the previous layer's quantiser leaves it
    x = torch.randint(-60, 61, (2, 13, 11, C), generator=g).float() / 16.0
    ho, wo = _out_hw(k, s)
    gy = torch.randn(2, ho, wo, C, generator=g)
    xs = x.cuda().requires_grad_(training)
    x64 = _nchw(x).double().requires_grad_(training)
    y64, leaves, rm64, rv64 = _layer64(c, x64, training, p)
    y = c(xs)
    y64 = y64.permute(0, 2, 3, 1)
    if not training:
        assert torch.equal(y.double().cpu(), y64.detach()), float((y.double().cpu() - y64).abs().max())
        return
    y.backward(gy.cuda())
    y64.backward(gy.double())
    ours = dict(weight=c.weight.grad, gamma=c.gamma.grad, beta=c.beta.grad, wscale=c.weight_quantizer.scale.grad,
                ascale=c.activation_quantizer.scale.grad)
    errs = {n: _rel(ours[n], leaves[n].grad) for n in ours}
    errs["x"] = _rel(xs.grad, x64.grad.permute(0, 2, 3, 1))
    errs["running"] = max(_rel(c.running_mean, rm64), _rel(c.running_var, rv64))
    codes_off = float((y.detach().double().cpu() - y64.detach()).abs().gt(0).double().mean())
    print("\n[tpsq depthwise C=%d k=%d s=%d %s %s] codes off %.3g %s" % (C, k, s, act, regime, codes_off,
                                                                       " ".join("%s=%.2g" % kv for kv in errs.items())))
    assert float(c.step) == {"first_step": 1, "before_freeze": 11, "after_freeze": c.freeze_step}[regime]
    assert float(c.first_bn) == 1
    assert max(errs.values()) < 1e-4, errs


# ---- against the reference's own run ----------------------------------------------------------------------------------
LAYERS = (13, 17, 27, 30, 60)


def test_tpsq_depthwise_layers_teacher_forced():
    """Five depthwise layers (5x5 stride 2 and 1 with relu6, 3x3 stride 2 and 1 with h_swish, the 960-channel 5x5) on
    the REFERENCE's own input tensor and output gradient of that layer, under the gates of
    test_gpu_qat.py::test_qat_layers_teacher_forced"""
    g = golden("yolov3-mobilenet_64_qat2_layers")
    qm = _model().train()
    worst = {"y_frac_off": 0.0, "y_max_lsb": 0.0, "gx": 0.0, "gw": 0.0, "ggamma": 0.0, "gbeta": 0.0, "stats": 0.0}
    for i in LAYERS:
        c = qm.module_list[i][0]
        x = torch.from_numpy(g["L%d.x" % i]).permute(0, 2, 3, 1).contiguous().cuda().requires_grad_(True)
        y = c(x)
        ref_y = torch.from_numpy(g["L%d.y" % i]).permute(0, 2, 3, 1)
        for n, b in c.named_buffers():
            key = "L%d.buf.%s" % (i, n)
            if key in g.files and n.endswith(("scale", "step", "first_bn")):
                assert float(b.reshape(-1)[0]) == float(g[key].reshape(-1)[0]), (i, n, float(b.reshape(-1)[0]), g[key])
            if key in g.files and n.endswith(("running_mean", "running_var")):
                r = torch.from_numpy(g[key])
                worst["stats"] = max(worst["stats"], float((b.cpu() - r).abs().max() / r.abs().max().clamp(min=1e-6)))
        for n, p_ in c.named_parameters():
            key = "L%d.par.%s" % (i, n)
            if key in g.files:       # TPSQ scale parameters after the Search_Pow2 snap
                assert float(p_.detach().reshape(-1)[0]) == float(g[key].reshape(-1)[0]), (i, n)
        d = (y.detach().cpu() - ref_y).abs()
        lsb = float(ref_y.abs()[ref_y.abs() > 0].min())
        worst["y_frac_off"] = max(worst["y_frac_off"], float((d > 0.25 * lsb).float().mean()))
        worst["y_max_lsb"] = max(worst["y_max_lsb"], float(d.max()) / lsb)
        y.backward(torch.from_numpy(g["L%d.gy" % i]).permute(0, 2, 3, 1).contiguous().cuda())
        rgx = torch.from_numpy(g["L%d.gx" % i]).permute(0, 2, 3, 1)
        worst["gx"] = max(worst["gx"], float((x.grad.cpu() - rgx).norm() / rgx.norm()))
        for n, p_ in c.named_parameters():
            key = "L%d.grad.%s" % (i, n)
            slot = {"weight": "gw", "gamma": "ggamma", "beta": "gbeta"}.get(n)
            if key not in g.files or slot is None:
                continue
            assert p_.grad is not None, (i, n)
            ref = torch.from_numpy(g[key])
            worst[slot] = max(worst[slot], float((p_.grad.detach().cpu() - ref).norm() / ref.norm().clamp(min=1e-12)))
    print("\n[tpsq depthwise layers, teacher forced] %s" % " ".join("%s=%.3g" % kv for kv in worst.items()))
    assert worst["y_frac_off"] < 5e-3 and worst["y_max_lsb"] <= 2.0
    assert worst["stats"] < 1e-4
    assert worst["gx"] < 5e-3 and worst["gw"] < 1e-3 and worst["ggamma"] < 1e-3 and worst["gbeta"] < 1e-5


def _step(qm):
    from utils import utils as my_utils
    x = orc.synth_images(2, 64, 64, seed=0).cuda()
    t = orc.synth_targets(2, 6, 80, seed=1).cuda()
    pred, _ = qm(x)
    loss, items = my_utils.compute_loss(pred, t, qm)
    loss.backward()
    torch.cuda.synchronize()
    return pred, items


def test_mobilenet_tpsq_training_step_and_eval_match_reference():
    """the gates of test_gpu_qat_mobilenet.py::test_mobilenet_qat_training_step_and_eval_match_reference"""
    g = golden("yolov3-mobilenet_64_qat2")
    qm = _model().train()
    pred, items = _step(qm)
    items_rel = float((np.abs(items.detach().cpu().numpy() - g["items"]) / np.abs(g["items"])).max())
    params = dict(qm.named_parameters())
    names = [str(n) for n in g["grad_names"]]
    ref = dict(zip(names, g["grad_norms"]))
    missing = [k for k in names if params[k].grad is None]
    floor = 1e-3 * float(np.median(list(ref.values())))
    rel = {k: abs(float(params[k].grad.norm()) - v) / max(v, floor) for k, v in ref.items() if params[k].grad is not None}
    dw_rel = [v for k, v in rel.items() if '.DepthWise2d.' in k]
    sd = qm.state_dict()
    sn, sv = [str(n) for n in g["scale_names"]], g["scale_values"]
    diff = [k for k, v in zip(sn, sv) if abs(float(sd[k].reshape(-1)[0]) - float(v)) > 1e-6 * abs(float(v))]
    i0 = next(i for i, d in enumerate(qm.module_defs) if d['type'] == 'depthwise')
    first = {n: float((sd['module_list.%d.DepthWise2d.%s' % (i0, n)].cpu() -
                       torch.from_numpy(g['state::module_list.%d.DepthWise2d.%s' % (i0, n)])).abs().max())
             for n in ('running_mean', 'running_var')}
    counters = [k for k in g.files if k.startswith('state::') and k.endswith(('.step', '.first_bn'))]
    counters_off = [k for k in counters if not torch.equal(sd[k[7:]].cpu(), torch.from_numpy(g[k]))]
    print("\n[yolov3-mobilenet tpsq train step vs reference] loss items rel %.3g | grad-norm rel median %.3g worst %.3g "
          "(depthwise median %.3g, %d params without grad) | scales differing %d of %d | first depthwise running stats "
          "abs %s | %d step / first_bn buffers" % (items_rel, np.median(list(rel.values())), max(rel.values()),
                                                  np.median(dw_rel), len(missing), len(diff), len(sn), first,
                                                  len(counters)))
    qm.eval()
    with torch.no_grad():
        io, p, _ = qm(orc.synth_images(2, 64, 64, seed=5).cuda())
    ref_io = torch.from_numpy(g["eval_io"])
    close = float(torch.isclose(io.cpu(), ref_io, rtol=2e-2, atol=2e-2).float().mean())
    print("[yolov3-mobilenet tpsq eval after the step] fraction of io within 2e-2: %.4f" % close)
    assert not missing
    assert items_rel < 0.1
    assert np.median(list(rel.values())) < 0.5
    assert len(diff) <= 0.12 * len(sn)
    assert max(first.values()) < 1e-4
    assert counters and not counters_off, counters_off[:5]
    assert torch.isfinite(io).all()


def test_mobilenet_tpsq_step_is_deterministic():
    grads = []
    for _ in range(2):
        qm = _model().train()
        _step(qm)
        grads.append({k: p.grad.detach().clone() for k, p in qm.named_parameters() if p.grad is not None})
    assert grads[0].keys() == grads[1].keys()
    bad = [k for k in grads[0] if not torch.equal(grads[0][k], grads[1][k])]
    assert not bad, bad[:5]


def test_mobilenet_tpsq_flat_optimizer_step():
    """FlatDataParallel + train.py's quantized=2 optimiser (Adam; pg3 holds the TPSQ scale parameters)"""
    from b200yolo.optim import make_optimizer
    from b200yolo.parallel import FlatDataParallel
    from optim_ref import HYP
    from utils import utils as my_utils
    dp = FlatDataParallel(_model().train())
    opt = make_optimizer(dp, dict(dp.module.hyp, **HYP), quantized=2)
    pred, _ = dp(orc.synth_images(2, 64, 64, seed=0).cuda())
    loss, _ = my_utils.compute_loss(pred, orc.synth_targets(2, 6, 80, seed=1).cuda(), dp.module)
    loss.backward()
    dws = [dp.module.module_list[i][0] for i, d in enumerate(dp.module.module_defs) if d['type'] == 'depthwise']
    tracked = {}
    for j, c in enumerate(dws):
        for n, t in (("weight", c.weight), ("wscale", c.weight_quantizer.scale), ("ascale", c.activation_quantizer.scale)):
            tracked["%d.%s" % (j, n)] = (t, t.detach().clone())
    opt.step()
    torch.cuda.synchronize()
    assert torch.isfinite(dp.flat_param).all()
    moved = {k: not torch.equal(t.detach(), before) for k, (t, before) in tracked.items()}
    assert all(v for k, v in moved.items() if k.endswith("weight")), moved
    assert all(v for k, v in moved.items() if k.endswith("scale")), moved
