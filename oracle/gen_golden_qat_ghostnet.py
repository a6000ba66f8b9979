"""Golden fixtures for the QAT graphs of yolov3-ghost: run the REFERENCE's own model on CPU for ONE training step
(forward, compute_loss, backward) at 64x64, batch 2, then an eval forward, for google QAT (quantized=1) with
shortcut_way 1 and 2 and for TPSQ (quantized=2).

Every GhostNet [convolutional] block, the depthwise cheap operations (groups=C, 3x3 and 5x5, strides 1 and 2) included,
is one quantised BN-folded layer of the mode (models.py:28-115); [se] stays the float SE; routes are
QuantizedFeatureConcat in both modes, shortcuts QuantizedShortcut_min / _max under quantized=1 and the plain Shortcut
under quantized=2.  The cfg is b200yolo.cfggen's yolov3-ghost, checked here against the reference's own cfg file.
Output: tests/golden/yolov3-ghost_64_qat1.npz (keys prefixed 'sw1.' and 'sw2.') and tests/golden/yolov3-ghost_64_qat2.npz.
Run here only."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("B2Y_REFERENCE_ROOT", "/root/reference")
PKG = os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200")
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "mpl_stub"))
os.chdir(REF)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import models as ref_models  # noqa: E402
from utils import utils as ru  # noqa: E402
from utils.parse_config import parse_model_cfg  # noqa: E402

sys.path.insert(0, HERE)
import darknet_oracle as orc  # noqa: E402

STEPS = 100
CFG = "cfg/yolov3-ghostnet/yolov3-ghost-coco.cfg"


def check_cfggen():
    """b200yolo.cfggen's yolov3-ghost parses to the reference cfg's layer definitions ([net] aside)"""
    import importlib.util
    import tempfile
    spec = importlib.util.spec_from_file_location("cfggen", os.path.join(PKG, "b200yolo", "cfggen.py"))
    cfggen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cfggen)
    with tempfile.TemporaryDirectory() as d:
        ours = parse_model_cfg(cfggen.write_cfg("yolov3-ghost", d))[1:]
    ref = parse_model_cfg(CFG)[1:]
    norm = lambda b: {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in b.items()}  # noqa: E731
    assert [norm(b) for b in ours] == [norm(b) for b in ref]


def load_synth(qm):
    """Quantised convs get the float model's synthetic conv weights, and its BatchNorm2d weight / bias as gamma / beta
    (running statistics stay zero: the first step seeds them); the float SE modules take theirs unchanged."""
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
        elif '.se.' in k and k in sd:
            new[k] = sd[k]
        else:
            new[k] = v
    qm.load_state_dict(new)


def run(quantized, shortcut_way):
    torch.manual_seed(0)
    qm = ref_models.Darknet(CFG, quantized=quantized, a_bit=8, w_bit=8, shortcut_way=shortcut_way, steps=STEPS)
    load_synth(qm)
    qm.nc, qm.gr, qm.hyp = 80, 1.0, dict(orc.DEFAULT_HYP)
    out = {"tree": np.array(["%d %s %s" % (i, n, c.__class__.__name__) for i, m in enumerate(qm.module_list)
                             for n, c in m.named_children()]),
           "state_keys": np.array(list(qm.state_dict().keys())),
           "param_names": np.array([n for n, _ in qm.named_parameters()])}
    B, S = 2, 64
    qm.train()
    pred, _ = qm(orc.synth_images(B, S, S, seed=0))
    loss, items = ru.compute_loss(pred, orc.synth_targets(B, 6, 80, seed=1), qm)
    loss.backward()
    out["items"], out["loss"] = items.numpy(), loss.detach().numpy()
    named = {k: p for k, p in qm.named_parameters() if p.grad is not None}
    out["grad_names"] = np.array(list(named))
    out["grad_norms"] = np.array([float(p.grad.norm()) for p in named.values()], dtype=np.float64)
    sd = qm.state_dict()
    for k, v in sd.items():
        # copies: the eval forward below must not reach the recorded state
        if k.endswith(('running_mean', 'running_var')):
            out["state::" + k] = v.detach().numpy().copy()
    # the step counters of the layers and quantisers and the first_bn flags, one array (the quantisers' step counters
    # advance in place in the eval forward below)
    counters = {k: float(v.reshape(-1)[0]) for k, v in sd.items() if k.endswith(('.step', '.first_bn'))}
    out["counter_names"] = np.array(list(counters))
    out["counter_values"] = np.array(list(counters.values()), dtype=np.float64)
    all_scales = {k: float(v.detach().reshape(-1)[0]) for k, v in sd.items() if k.endswith('.scale') and v.numel() == 1}
    out["scale_names"] = np.array(list(all_scales))
    out["scale_values"] = np.array(list(all_scales.values()), dtype=np.float64)
    qm.eval()
    with torch.no_grad():
        io, p, _ = qm(orc.synth_images(B, S, S, seed=5))
    out["eval_io"] = io.numpy()
    for i, pi in enumerate(p):
        out["eval_p%d" % i] = pi.numpy()
    print("yolov3-ghost quantized=%d shortcut_way=%d loss" % (quantized, shortcut_way), float(loss), items.tolist(),
          "n scales", len(all_scales), "eval io mean", float(io.abs().mean()))
    return out


def main():
    torch.set_num_threads(8)
    check_cfggen()
    gold = os.path.join(ROOT, "tests", "golden")
    qat1 = {}
    for sw in (1, 2):
        qat1.update({"sw%d.%s" % (sw, k): v for k, v in run(1, sw).items()})
    np.savez_compressed(os.path.join(gold, "yolov3-ghost_64_qat1.npz"), **qat1)
    np.savez_compressed(os.path.join(gold, "yolov3-ghost_64_qat2.npz"), **run(2, 1))


if __name__ == "__main__":
    main()
