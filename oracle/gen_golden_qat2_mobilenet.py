"""Golden fixtures for the TPSQ (quantized=2, shortcut_way=1) graph of yolov3-mobilenet: run the REFERENCE's own model on
CPU for ONE training step (forward, compute_loss, backward) at 64x64, batch 2, then an eval forward.

Under quantized=2 every [depthwise] block is one TPSQ_BNFold_QuantizedConv2d_For_FPGA(groups=C) named DepthWise2d
(models.py:140-155), with the BN fold, the power-of-two weight / activation quantisers and the bias quantiser of the dense
TPSQ layer.  [se] stays the float SE.  Module-boundary tensors of five depthwise layers are captured by hooks for the
teacher-forced layer test (3x3 and 5x5, strides 1 and 2, relu6 and h_swish, and the widest, 960-channel layer).
Output: tests/golden/yolov3-mobilenet_64_qat2.npz and tests/golden/yolov3-mobilenet_64_qat2_layers.npz.   Run here only."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("B2Y_REFERENCE_ROOT", "/root/reference")
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "mpl_stub"))
os.chdir(REF)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import models as ref_models  # noqa: E402
from utils import utils as ru  # noqa: E402

sys.path.insert(0, HERE)
import darknet_oracle as orc  # noqa: E402

STEPS = 100
CFG = "cfg/yolov3-mobilenet/yolov3-mobilenet-coco.cfg"
# [depthwise] layers: 13 5x5/2 relu6 (72), 17 5x5/1 relu6 (120), 27 3x3/2 h_swish (240), 30 3x3/1 h_swish (200),
# 60 5x5/1 h_swish (960, the widest)
LAYERS = (13, 17, 27, 30, 60)


def load_synth(qm):
    """Quantised Conv2d / DepthWise2d modules get the float model's synthetic weights, and its BatchNorm2d weight / bias
    as gamma / beta (running statistics stay zero: the first step seeds them); the float SE modules take theirs
    unchanged."""
    sd = orc.synth_state_dict(ref_models.Darknet(CFG).state_dict(), 0)
    new = {}
    for k, v in qm.state_dict().items():
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


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    qm = ref_models.Darknet(CFG, quantized=2, a_bit=8, w_bit=8, shortcut_way=1, steps=STEPS)
    load_synth(qm)
    qm.nc, qm.gr, qm.hyp = 80, 1.0, dict(orc.DEFAULT_HYP)
    out = {"tree": np.array(["%d %s %s" % (i, n, c.__class__.__name__) for i, m in enumerate(qm.module_list)
                             for n, c in m.named_children()]),
           "state_keys": np.array(list(qm.state_dict().keys())),
           "param_names": np.array([n for n, _ in qm.named_parameters()])}
    B, S = 2, 64
    qm.train()
    x = orc.synth_images(B, S, S, seed=0)
    t = orc.synth_targets(B, 6, 80, seed=1)
    lay = {}

    def fwd_hook(i):
        def f(m, inp, out_):
            lay["L%d.x" % i] = inp[0].detach().numpy().copy()
            lay["L%d.y" % i] = out_.detach().numpy().copy()
        return f

    def bwd_hook(i):
        def f(m, gin, gout):
            if gin[0] is not None:
                lay["L%d.gx" % i] = gin[0].detach().numpy().copy()
            lay["L%d.gy" % i] = gout[0].detach().numpy().copy()
        return f

    for i in LAYERS:
        assert qm.module_defs[i]['type'] == 'depthwise'
        qm.module_list[i][0].register_forward_hook(fwd_hook(i))
        qm.module_list[i][0].register_full_backward_hook(bwd_hook(i))
    pred, _ = qm(x)
    loss, items = ru.compute_loss(pred, t, qm)
    loss.backward()
    for i in LAYERS:
        c = qm.module_list[i][0]
        for n, p_ in c.named_parameters():
            if p_.grad is not None:
                lay["L%d.grad.%s" % (i, n)] = p_.grad.numpy().copy()
        for n, b_ in c.named_buffers():
            if n.endswith(("scale", "running_mean", "running_var", "batch_mean", "batch_var", "min_val", "max_val",
                           "step", "first_bn")):
                lay["L%d.buf.%s" % (i, n)] = b_.detach().numpy().copy()
        for n, p_ in c.named_parameters():
            if n.endswith("scale"):
                lay["L%d.par.%s" % (i, n)] = p_.detach().numpy().copy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "yolov3-mobilenet_64_qat2_layers.npz"), **lay)
    out["items"], out["loss"] = items.numpy(), loss.detach().numpy()
    named = {k: p for k, p in qm.named_parameters() if p.grad is not None}
    out["grad_names"] = np.array(list(named))
    out["grad_norms"] = np.array([float(p.grad.norm()) for p in named.values()], dtype=np.float64)
    sd = qm.state_dict()
    for k, v in sd.items():
        if k.endswith(('running_mean', 'running_var', '.scale', 'min_val', 'max_val', 'step', 'first_bn')) and \
                v.numel() <= 1024:
            out["state::" + k] = v.detach().numpy()
    all_scales = {k: float(v.detach().reshape(-1)[0]) for k, v in sd.items() if k.endswith('.scale') and v.numel() == 1}
    out["scale_names"] = np.array(list(all_scales))
    out["scale_values"] = np.array(list(all_scales.values()), dtype=np.float64)
    qm.eval()
    with torch.no_grad():
        io, p, _ = qm(orc.synth_images(B, S, S, seed=5))
    out["eval_io"] = io.numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "yolov3-mobilenet_64_qat2.npz"), **out)
    print("yolov3-mobilenet qat2 loss", float(loss), items.tolist(), "n scales", len(all_scales),
          "eval io mean", float(io.abs().mean()))


if __name__ == "__main__":
    main()
