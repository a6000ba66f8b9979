"""Generate the fixtures of the wide-head and focal-loss tests by RUNNING THE REFERENCE ITSELF (the checkout that
gen_golden.py imports, on the CPU) with the recipe of gen_golden.py: synthetic weights of seed 0, synth_images /
synth_targets, HYP.  It writes new files only:

    tests/golden/heads_cfg.json                      the reference's parse of cfg/yolov2/yolov2{,-tiny}.cfg
    tests/golden/yolov2-tiny_96_eval.npz             eval forward at 2 x 96^2 (one 425-wide head)
    tests/golden/yolov2-tiny_128_train.npz           training step at 4 x 128^2
    tests/golden/yolov3-tiny-nc100_128_train.npz     training step of the 100-class yolov3-tiny (315-wide heads)
    tests/golden/focal_case.npz                      compute_loss with hyp['fl_gamma'] > 0

    python oracle/gen_golden_heads.py
"""
import importlib.util
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.dont_write_bytecode = True
sys.path.insert(0, HERE)
import gen_golden as G  # noqa: E402  (puts the reference on sys.path and chdirs into it)
from gen_golden import GOLD, orc, ref_models, ref_utils  # noqa: E402
import gen_golden_cfg  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"))
from b200yolo import cfggen  # noqa: E402

V2_CFGS = {"yolov2": "cfg/yolov2/yolov2.cfg", "yolov2-tiny": "cfg/yolov2/yolov2-tiny.cfg"}
GAMMAS = {"g15": 1.5, "g05": 0.5}


def build(cfg, seed=0):
    m = ref_models.Darknet(cfg)
    m.load_state_dict(orc.synth_state_dict(m.state_dict(), seed))
    return m


def train_fixture(m, nc, tag):
    """gen_golden.py's training-step fixture: items, p*, gradient norms, full gradients of the first two and last four
    parameters (fp16 beyond 2^18 elements), running statistics."""
    m.train()
    G.attach_hyp(m, nc)
    x = orc.synth_images(4, 128, 128, seed=0)
    t = orc.synth_targets(4, 6, nc, seed=1)
    pred, _ = m(x)
    loss, items = ref_utils.compute_loss(pred, t, m)
    loss.backward()
    sd = m.state_dict()
    out = {"loss": loss.detach().numpy(), "items": items.numpy()}
    for i, pi in enumerate(pred):
        out["p%d" % i] = pi.detach().numpy()
    names, norms = [], []
    for k, prm in m.named_parameters():
        names.append(k)
        norms.append(float(prm.grad.norm()) if prm.grad is not None else -1.0)
    out["grad_names"] = np.array(names)
    out["grad_norms"] = np.array(norms, dtype=np.float64)
    keep = [k for k in names if k.startswith("module_list.0.") or k.startswith("module_list.1.")]
    keep += names[-4:]
    for k in keep:
        grad = dict(m.named_parameters())[k].grad.numpy()
        # the 425 x 1024 head of yolov2-tiny: stored rounded to fp16 (2^-11 relative per element, far below the 2 %
        # element-wise gate of its test), which keeps the fixture under 1 MB
        out["grad::" + k] = grad.astype(np.float16) if grad.size > (1 << 18) else grad
    bn_keys = [k for k in sd if k.endswith("running_mean") or k.endswith("running_var")]
    for k in bn_keys[:4] + bn_keys[-2:]:
        out["stat::" + k] = sd[k].numpy()
    np.savez_compressed(os.path.join(GOLD, tag + ".npz"), **out)
    print(tag, "loss", float(loss), items.tolist())


def loss_with_grad(m, preds, t, gamma):
    m.hyp['fl_gamma'] = gamma
    ps = [p.detach().clone().requires_grad_(True) for p in preds]
    loss, items = ref_utils.compute_loss(ps, t, m)
    loss.backward()
    return items.numpy(), [p.grad.numpy() for p in ps]


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref = os.getcwd()
    # ---- the reference's parse of its yolov2 cfgs ---------------------------------------------------------------
    spec = importlib.util.spec_from_file_location("ref_parse_config", os.path.join(ref, "utils", "parse_config.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    layers = {name: [{k: gen_golden_cfg._plain(d[k]) for k in gen_golden_cfg.KEYS if k in d}
                     for d in mod.parse_model_cfg(rel)[1:]] for name, rel in V2_CFGS.items()}
    with open(os.path.join(GOLD, "heads_cfg.json"), "w") as f:
        json.dump(layers, f, sort_keys=True, separators=(",", ":"))

    # ---- yolov2-tiny: eval forward and training step ------------------------------------------------------------
    m = build(V2_CFGS["yolov2-tiny"]).eval()
    with torch.no_grad():
        io, p, _ = m(orc.synth_images(2, 96, 96, seed=3))
    np.savez_compressed(os.path.join(GOLD, "yolov2-tiny_96_eval.npz"), io=io.numpy(),
                        **{"p%d" % i: t.numpy() for i, t in enumerate(p)})
    print("yolov2-tiny_96_eval", tuple(io.shape))
    train_fixture(build(V2_CFGS["yolov2-tiny"]), 80, "yolov2-tiny_128_train")

    # ---- yolov3-tiny with 100 classes: 3 * 105 = 315 head filters ------------------------------------------------
    with tempfile.TemporaryDirectory() as d:
        cfg = os.path.join(d, "yolov3-tiny-nc100.cfg")
        with open(cfg, "w") as f:
            f.write(cfggen.cfg_text("yolov3-tiny", classes=100))
        m = build(cfg)
    train_fixture(m, 100, "yolov3-tiny-nc100_128_train")

    # ---- focal loss ---------------------------------------------------------------------------------------------
    # loss_case of gen_golden.py (yolov3 anchors, grids 2/4/8 at B=3) at two gammas
    m = build(G.CFGS["yolov3"])
    G.attach_hyp(m)
    g = torch.Generator().manual_seed(7)
    preds = [torch.randn(3, 3, s, s, 85, generator=g) for s in (2, 4, 8)]
    for j, s in zip(m.yolo_layers, (2, 4, 8)):
        m.module_list[j].create_grids((s, s))
    t = orc.synth_targets(3, 10, 80, seed=5)
    out = {"targets": t.numpy()}
    for i, p in enumerate(preds):
        out["p%d" % i] = p.numpy()
    for key, gamma in GAMMAS.items():
        items, dps = loss_with_grad(m, preds, t, gamma)
        out["items_" + key] = items
        for i, d in enumerate(dps):
            out["dp%d_%s" % (i, key)] = d
    # saturated logits: every objectness / class logit set to +-30 (sigma rounds to exactly 1 / 0 in fp32)
    sat = [p.clone() for p in preds]
    for p in sat:
        p[..., 4:] = torch.where(p[..., 4:] > 0, torch.tensor(30.0), torch.tensor(-30.0))
    items, dps = loss_with_grad(m, sat, t, 1.5)
    out["items_sat"] = items
    for i, (p, d) in enumerate(zip(sat, dps)):
        out["sat_p%d" % i] = p.numpy()
        out["dp%d_sat" % i] = d
    # several targets in one cell (yolov3-tiny anchors, grids 2/4): the last match owns tobj
    m = build(G.CFGS["yolov3-tiny"])
    G.attach_hyp(m)
    for j, s in zip(m.yolo_layers, (2, 4)):
        m.module_list[j].create_grids((s, s))
    g = torch.Generator().manual_seed(9)
    dup = [torch.randn(2, 3, s, s, 85, generator=g) for s in (2, 4)]
    td = torch.tensor([[0, 3, 0.26, 0.26, 0.3, 0.4], [0, 5, 0.27, 0.27, 0.3, 0.4], [0, 7, 0.27, 0.26, 0.31, 0.41],
                       [1, 1, 0.8, 0.8, 0.2, 0.1]], dtype=torch.float32)
    items, dps = loss_with_grad(m, dup, td, 1.5)
    out["dup_targets"] = td.numpy()
    out["items_dup"] = items
    for i, (p, d) in enumerate(zip(dup, dps)):
        out["dup_p%d" % i] = p.numpy()
        out["dp%d_dup" % i] = d
    np.savez_compressed(os.path.join(GOLD, "focal_case.npz"), **out)
    print("focal case", out["items_g15"].tolist(), out["items_g05"].tolist(), out["items_sat"].tolist(),
          out["items_dup"].tolist())
    print("done ->", GOLD)


if __name__ == "__main__":
    main()
