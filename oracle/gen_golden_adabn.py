"""Generate tests/golden/pruned_adabn_case.npz by RUNNING THE REFERENCE (CPU) through the adaptive-BatchNorm step of its
EagleEye pruning search (EagleEye_normal_prune.py:123-130): a candidate sub-network in train mode, forwards under
torch.no_grad() that only refresh the BatchNorm running statistics, then the evaluation forward.

    python oracle/gen_golden_adabn.py

The candidates are the compact models of tests/golden/pruned_case.npz (oracle/gen_golden_pruned.py: yolov3-tiny 96 px,
yolov3 64 px, yolov3-mobilenet 128 px), rebuilt from that fixture with the reference's Darknet: the stock cfg with the
kept widths, and the loose model's synthetic parameters (orc.synth_state_dict, seed 0) cut down to the kept output and
input channels.  The rebuild is checked against the per-tensor sums the pruned fixture stores.

Per case: p of each of the three recalibration batches (orc.synth_images(4, size, size, seed 11 / 12 / 13)), every
BatchNorm's running_mean / running_var / num_batches_tracked afterwards, and the eval io for
orc.synth_images(2, size, size, seed=5) after the recalibration.  To keep the file small, p and io are stored as
rows(t): every step-th output row of each image ([B, rows, no] with step = ceil(rows / 16)); the tests take the same rows.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_golden_pruned as gp  # noqa: E402  (puts the reference first on sys.path and changes into it)

ref_models, orc = gp.ref_models, gp.orc

SEEDS = (11, 12, 13)
BATCH = 4
ROWS = 16


def rows(t):
    """[B, ..., no] -> [B, <= ROWS, no]: every step-th output row of each image"""
    t = t.reshape(t.shape[0], -1, t.shape[-1])
    return t[:, ::-(-t.shape[1] // ROWS)]


def compact_model(g, name, cfg, size):
    """the compact model of the pruned fixture, in the reference's Darknet"""
    loose = ref_models.Darknet(cfg, img_size=(size, size))
    loose_sd = orc.synth_state_dict(loose.state_dict(), 0)
    defs = [loose.hyperparams.copy()] + [dict(d) for d in loose.module_defs]
    for i, w in json.loads(str(g[name + ":widths_json"])).items():
        defs[int(i) + 1]['filters'] = str(w)
    model = ref_models.Darknet(defs, img_size=(size, size))
    sd = {}
    for k, v in model.state_dict().items():
        i = int(k.split('.')[1])
        t = loose_sd[k]
        kept = "%s:out%d" % (name, i)
        o = torch.from_numpy(g[kept].astype(np.int64)) if kept in g else None
        if '.se.fc.0.' in k:
            t = t[:v.shape[0]][:, o]
        elif '.se.fc.2.' in k:
            t = t[o][:, :v.shape[1]]
        elif t.dim() > 0:
            if o is not None:
                t = t[o]
            if t.dim() == 4 and "%s:in%d" % (name, i) in g:
                t = t[:, torch.from_numpy(g["%s:in%d" % (name, i)].astype(np.int64))]
        sd[k] = t.clone()
    model.load_state_dict(sd)
    names = sorted(sd)
    assert names == [str(s) for s in g[name + ":sd_names"]]
    np.testing.assert_allclose([float(sd[k].double().sum()) for k in names], g[name + ":sd_sums"], rtol=1e-12)
    return model


def run_case(g, name, cfg, size):
    model = compact_model(g, name, cfg, size)
    out = {}
    model.train()
    with torch.no_grad():
        for b, seed in enumerate(SEEDS):
            yolo_out, _ = model(orc.synth_images(BATCH, size, size, seed=seed))
            for j, p in enumerate(yolo_out):
                out["p%d_%d" % (b, j)] = rows(p).numpy()
    for k, v in model.state_dict().items():
        if k.endswith(('running_mean', 'running_var', 'num_batches_tracked')):
            out["stat::" + k] = v.numpy()
    model.eval()
    with torch.no_grad():
        out["io"] = rows(model(orc.synth_images(2, size, size, seed=5))[0]).numpy()
    print("%s %dpx: %d BatchNorms recalibrated over %d batches of %d" %
          (name, size, sum(k.endswith('running_mean') for k in out if k.startswith('stat::')), len(SEEDS), BATCH))
    return {"%s:%s" % (name, k): v for k, v in out.items()}


def main():
    torch.set_num_threads(1)        # the reference's CPU reductions in a fixed order: the file is reproducible
    g = dict(np.load(os.path.join(gp.ROOT, "tests", "golden", "pruned_case.npz")))
    out = {"cases": np.array(json.dumps([[n, s] for n, _, s in gp.CASES])),
           "seeds": np.array(SEEDS), "batch": np.array(BATCH)}
    for name, cfg, size in gp.CASES:
        out.update(run_case(g, name, cfg, size))
    np.savez_compressed(os.path.join(gp.ROOT, "tests", "golden", "pruned_adabn_case.npz"), **out)


if __name__ == "__main__":
    main()
