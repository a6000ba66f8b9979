"""Golden fixture for the google QAT (quantized=1, shortcut_way=1) graph of yolov3-mobilenet: run the REFERENCE's own
model on CPU for ONE training step (forward, compute_loss, backward) at 64x64, batch 2, then an eval forward.

Under quantized=1 the reference builds every [depthwise] block as a plain nn.Conv2d(groups=C) + BatchNorm2d +
activation (models.py:115-197: the `else` of the quantized 2 / 3 test also runs for 1 and replaces 'DepthWise2d'), and
[se] as the float SE layer.  The module tree is recorded so the tests can compare ours against it.
Output: tests/golden/yolov3-mobilenet_64_qat1.npz.   Run here only."""
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


def load_synth(qm):
    """QAT convs get the float model's synthetic conv / BatchNorm values (gamma, beta on the conv module, running
    statistics left at their initial values); the float depthwise / BatchNorm / SE modules take them unchanged."""
    sd = orc.synth_state_dict(ref_models.Darknet(CFG).state_dict(), 0)
    new = {}
    for k, v in qm.state_dict().items():
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


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    qm = ref_models.Darknet(CFG, quantized=1, a_bit=8, w_bit=8, shortcut_way=1, steps=STEPS)
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
    pred, _ = qm(x)
    loss, items = ru.compute_loss(pred, t, qm)
    loss.backward()
    out["items"], out["loss"] = items.numpy(), loss.detach().numpy()
    for i, pi in enumerate(pred):
        out["p%d" % i] = pi.detach().numpy()
    named = {k: p for k, p in qm.named_parameters() if p.grad is not None}
    out["grad_names"] = np.array(list(named))
    out["grad_norms"] = np.array([float(p.grad.norm()) for p in named.values()], dtype=np.float64)
    for k, p in named.items():
        if p.numel() <= 4096:
            out["grad::" + k] = p.grad.numpy()
    sd = qm.state_dict()
    for k, v in sd.items():
        if k.endswith(('running_mean', 'running_var', 'num_batches_tracked', '.scale', 'min_val', 'max_val',
                       'input_scale', 'step')) and v.numel() <= 4096:
            out["state::" + k] = v.detach().numpy()
    all_scales = {k: float(v.detach().reshape(-1)[0]) for k, v in sd.items() if k.endswith('.scale') and v.numel() == 1}
    out["scale_names"] = np.array(list(all_scales))
    out["scale_values"] = np.array(list(all_scales.values()), dtype=np.float64)
    qm.eval()
    with torch.no_grad():
        io, p, _ = qm(orc.synth_images(B, S, S, seed=5))
    out["eval_io"] = io.numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "yolov3-mobilenet_64_qat1.npz"), **out)
    print("yolov3-mobilenet qat1 loss", float(loss), items.tolist(), "n scales", len(all_scales),
          "eval io mean", float(io.abs().mean()))


if __name__ == "__main__":
    main()
