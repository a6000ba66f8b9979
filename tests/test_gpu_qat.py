"""GPU: quantisation-aware-training graphs (quantized=1 google QAT with shortcut_way=1, quantized=2 TPSQ; SURVEY 8a rows a22 /
a23) against fixtures produced by the reference itself (oracle/gen_golden_qat.py: ONE training step -- forward,
compute_loss, backward -- of yolov3 at 64x64, batch 2, then an eval forward).  The QAT layers run as module forwards
over NHWC tensors composed of the sm_90a kernels (b200yolo/qat.py)."""
import numpy as np
import pytest
import torch

from helpers import attach_hyp, cfg_path, golden, orc

pytestmark = pytest.mark.gpu

STEPS = 100


def _model(mode, name="yolov3"):
    import models
    fm = models.Darknet(cfg_path(name))
    sd = orc.synth_state_dict(fm.state_dict(), 0)
    qm = models.Darknet(cfg_path(name), quantized=mode, a_bit=8, w_bit=8, shortcut_way=1, steps=STEPS)
    with torch.no_grad():
        for i, m in enumerate(qm.module_list):
            pre = 'module_list.%d.' % i
            if m.__class__.__name__ == 'Sequential' and len(m) and hasattr(m[0], 'activation_quantizer'):
                c = m[0]
                c.weight.copy_(sd[pre + 'Conv2d.weight'])
                if (pre + 'BatchNorm2d.weight') in sd:
                    c.gamma.copy_(sd[pre + 'BatchNorm2d.weight'])
                    c.beta.copy_(sd[pre + 'BatchNorm2d.bias'])
                else:
                    c.bias.copy_(sd[pre + 'Conv2d.bias'])
    return attach_hyp(qm.cuda())


@pytest.mark.parametrize("name,mode,tag", [("yolov3", 1, "qat1"), ("yolov3", 2, "qat2"),
                                           ("yolov3-tiny", 1, "qat1"), ("yolov3-tiny", 2, "qat2")])
def test_qat_training_step_and_eval_match_reference(name, mode, tag):
    """yolov3: 75 QAT conv layers with quantised shortcuts / concats; yolov3-tiny: the max-pool (and zero-pad + max-pool)
    layers inside the QAT graphs (models.py:207-215)."""
    from utils import utils as my_utils
    g = golden("%s_64_%s" % (name, tag))
    qm = _model(mode, name).train()
    x = orc.synth_images(2, 64, 64, seed=0).cuda()
    t = orc.synth_targets(2, 6, 80, seed=1).cuda()
    pred, _ = qm(x)
    loss, items = my_utils.compute_loss(pred, t, qm)
    loss.backward()
    torch.cuda.synchronize()
    items_rel = float((np.abs(items.detach().cpu().numpy() - g["items"]) / np.abs(g["items"])).max())
    p_abs = max(float((pi.detach().cpu() - torch.from_numpy(g["p%d" % i])).abs().max()) for i, pi in enumerate(pred))
    p_rms = max(float((pi.detach().cpu() - torch.from_numpy(g["p%d" % i])).pow(2).mean().sqrt()) for i, pi in enumerate(pred))
    params = dict(qm.named_parameters())
    names = [str(n) for n in g["grad_names"]]
    ref = dict(zip(names, g["grad_norms"]))
    missing = [k for k in names if params[k].grad is None]
    floor = 1e-3 * float(np.median(list(ref.values())))
    rel = np.array([abs(float(params[k].grad.norm()) - v) / max(v, floor) for k, v in ref.items() if params[k].grad is not None])
    # quantiser scales after the step: powers of two -> exact equality expected (a fold computed from fp16-rounded
    # batch statistics may move a range across a power-of-two boundary in rare layers)
    sd = qm.state_dict()
    sn, sv = [str(n) for n in g["scale_names"]], g["scale_values"]
    diff = [(k, float(sd[k].reshape(-1)[0]), float(v)) for k, v in zip(sn, sv)
            if abs(float(sd[k].reshape(-1)[0]) - float(v)) > 1e-6 * abs(float(v))]
    stat = 0.0
    for k in g.files:
        if k.startswith("state::") and k.endswith(("running_mean", "running_var")):
            r = torch.from_numpy(g[k])
            stat = max(stat, float((sd[k[7:]].cpu() - r).abs().max() / r.abs().max().clamp(min=1e-6)))
    tag = "%s %s" % (name, tag)
    print("\n[%s train step vs reference] loss items rel %.3g | p abs %.3g rms %.3g | grad-norm rel median %.3g worst %.3g "
          "(%d params without grad) | scales differing %d of %d %s | running stats rel %.3g"
          % (tag, items_rel, p_abs, p_rms, np.median(rel), rel.max(), len(missing), len(diff), len(sn), diff[:3], stat))
    qm.eval()
    with torch.no_grad():
        io, p, _ = qm(orc.synth_images(2, 64, 64, seed=5).cuda())
    ref_io = torch.from_numpy(g["eval_io"])
    close = float(torch.isclose(io.cpu(), ref_io, rtol=2e-2, atol=2e-2).float().mean())
    print("[%s eval after the step] fraction of io within 2e-2: %.4f, max abs diff %.3g" % (tag, close, float((io.cpu() - ref_io).abs().max())))
    # End to end this 75-layer QAT network (batch-statistics fold on as few as 2x4x4 samples, 8-bit re-quantisation after
    # every layer) amplifies a single flipped code chaotically: the first block agrees with the reference to 5e-7 in the
    # batch statistics and in all but 0.02 % of the output codes, 86 % of the codes differ by layer 36 (tools/debug_qat.py).
    # The end-to-end gates are therefore statistical; the exact gates are per layer on the reference's own tensors
    # (test_qat_layers_teacher_forced below).
    assert not missing
    assert items_rel < 0.1
    assert np.median(rel) < 0.5
    assert len(diff) <= 0.12 * len(sn)


@pytest.mark.parametrize("mode,tag", [(1, "qat1"), (2, "qat2")])
def test_qat_layers_teacher_forced(mode, tag):
    """Five QAT conv layers (3x3 stride 2, 3x3, two 1x1, the bias-only head) run on the REFERENCE's own input tensor and
    output gradient of that layer (module-boundary tensors captured by hooks in oracle/gen_golden_qat.py): output values,
    quantiser scales, batch statistics, and the gradients w.r.t. the input, the weights and gamma / beta must match."""
    g = golden("yolov3_64_%s_layers" % tag)
    qm = _model(mode).train()
    worst = {"y_frac_off": 0.0, "y_max_lsb": 0.0, "gx": 0.0, "gw": 0.0, "ggamma": 0.0, "gbeta": 0.0, "stats": 0.0}
    for i in (5, 13, 39, 63, 81):
        c = qm.module_list[i][0]
        x = torch.from_numpy(g["L%d.x" % i]).permute(0, 2, 3, 1).contiguous().cuda().requires_grad_(True)
        y = c(x)
        ref_y = torch.from_numpy(g["L%d.y" % i]).permute(0, 2, 3, 1)
        a_scale = float(c.activation_quantizer.scale.detach().reshape(-1)[0]) if mode == 1 else None
        for n, b in c.named_buffers():
            key = "L%d.buf.%s" % (i, n)
            if key in g.files and n.endswith("scale"):
                assert float(b.reshape(-1)[0]) == float(g[key].reshape(-1)[0]), (i, n, float(b.reshape(-1)[0]), g[key])
            if key in g.files and n.endswith(("running_mean", "running_var")):
                r = torch.from_numpy(g[key])
                worst["stats"] = max(worst["stats"], float((b.cpu() - r).abs().max() / r.abs().max().clamp(min=1e-6)))
        for n, p_ in c.named_parameters():
            key = "L%d.par.%s" % (i, n)
            if key in g.files:       # TPSQ scale parameters after the Search_Pow2 snap
                assert float(p_.detach().reshape(-1)[0]) == float(g[key].reshape(-1)[0]), (i, n)
        d = (y.detach().cpu() - ref_y).abs()
        lsb = a_scale if a_scale else float(ref_y.abs()[ref_y.abs() > 0].min())
        worst["y_frac_off"] = max(worst["y_frac_off"], float((d > 0.25 * lsb).float().mean()))
        worst["y_max_lsb"] = max(worst["y_max_lsb"], float(d.max()) / lsb)
        gy = torch.from_numpy(g["L%d.gy" % i]).permute(0, 2, 3, 1).contiguous().cuda()
        y.backward(gy)
        if ("L%d.gx" % i) in g.files:
            rgx = torch.from_numpy(g["L%d.gx" % i]).permute(0, 2, 3, 1)
            worst["gx"] = max(worst["gx"], float((x.grad.cpu() - rgx).norm() / rgx.norm()))
        for n, p_ in c.named_parameters():
            key = "L%d.grad.%s" % (i, n)
            if key not in g.files or p_.grad is None:
                continue
            ref = torch.from_numpy(g[key])
            mine = p_.grad.detach().cpu()
            mine = mine if mine.shape == ref.shape else mine[:ref.shape[0]]
            err = float((mine - ref).norm() / ref.norm().clamp(min=1e-12))
            slot = "gw" if n == "weight" else ("ggamma" if n == "gamma" else ("gbeta" if n in ("beta", "bias") else None))
            if slot:
                worst[slot] = max(worst[slot], err)
    print("\n[%s layers, teacher forced] %s" % (tag, " ".join("%s=%.3g" % kv for kv in worst.items())))
    # y codes may be off by one LSB where a value sits on a rounding boundary; gx carries the bf16 store of the data
    # gradient (the printed maxima are the measured values)
    assert worst["y_frac_off"] < 5e-3 and worst["y_max_lsb"] <= 2.0
    assert worst["stats"] < 1e-4
    assert worst["gx"] < 5e-3 and worst["gw"] < 1e-3 and worst["ggamma"] < 1e-3 and worst["gbeta"] < 1e-5
