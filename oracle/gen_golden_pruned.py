"""Generate tests/golden/pruned_case.npz by RUNNING THE REFERENCE (CPU) on channel-pruned models, built the way its
pruning scripts build them (normal_prune.py:140-171, shortcut_prune.py): a BatchNorm-gamma mask per layer -> compact
module_defs with the kept widths -> Darknet(list) -> weights copied from the loose model with
utils/prune_utils.init_weights_from_loose_model.

    python oracle/gen_golden_pruned.py

Cases (batch 2, seeded synthetic weights and images):
  yolov3-tiny        96 px: widths 13, 3, 1, 37, 250, 100 (= 4 mod 8), 333, 77; the concat of layer 20 is [37 | 37]
  yolov3             64 px: every BatchNorm conv pruned to 30-95 %; the convs a shortcut adds share one mask (both
                     addends pruned alike, as shortcut / slim pruning does); the concat sources have odd widths
  yolov3-mobilenet  128 px: the same, and the depthwise and squeeze-excite layers keep the channels of the conv before
                     them (their weights are selected here: the reference's loose-model copy takes them whole)

Each case stores the kept widths, the kept output and input channels of every layer, per-tensor sums of the compact
state_dict and the reference's fp32 eval output for orc.synth_images(2, size, size, seed=5).  The loose model is the
stock cfg with orc.synth_state_dict(seed 0), which the tests rebuild from the generated cfgs, so they need neither the
reference checkout nor its cfg files.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("B2Y_REFERENCE_ROOT", "/root/reference")
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "mpl_stub"))
sys.path.insert(0, os.path.join(HERE, "terminaltables_stub"))
os.chdir(REF)

from copy import deepcopy  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

import models as ref_models  # noqa: E402  (the reference)
from utils import prune_utils as pu  # noqa: E402

sys.path.insert(0, HERE)
import darknet_oracle as orc  # noqa: E402

CASES = (("yolov3-tiny", "cfg/yolov3tiny/yolov3-tiny.cfg", 96),
         ("yolov3", "cfg/yolov3/yolov3.cfg", 64),
         ("yolov3-mobilenet", "cfg/yolov3-mobilenet/yolov3-mobilenet-coco.cfg", 128))
TINY_WIDTHS = {0: 13, 2: 3, 4: 1, 8: 37, 10: 250, 13: 100, 14: 333, 18: 37, 21: 77}


def jsonable(defs):
    return [{k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in d.items()} for d in defs]


def shortcut_groups(defs, cbl):
    """union of the convs whose outputs one shortcut adds (prune_utils.parse_module_defs2's pairing)"""
    parent = {i: i for i in cbl}

    def find(i):
        while parent[i] != i:
            i = parent[i]
        return i
    for i, d in enumerate(defs):
        if d['type'] == 'shortcut':
            j = i + int(d['from'][0])
            j = j if defs[j]['type'] == 'convolutional' else j - 1
            if i - 1 in parent and j in parent:
                parent[find(i - 1)] = find(j)
    return find


def keep_width(name, defs, i, rs):
    C = int(defs[i]['filters'])
    if name == "yolov3-tiny":
        return TINY_WIDTHS.get(i, C)
    k = max(1, int(round(C * rs.uniform(0.3, 0.95))))
    return k + 4 - k % 8 if C >= 16 and i % 5 == 0 else k    # some widths = 4 mod 8


def build_case(name, cfg, size):
    loose = ref_models.Darknet(cfg, img_size=(size, size))
    loose.load_state_dict(orc.synth_state_dict(loose.state_dict(), 0))
    defs = loose.module_defs
    CBL_idx, Other_idx, _ = pu.parse_module_defs(defs)
    find = shortcut_groups(defs, CBL_idx)
    rs = np.random.RandomState(7)
    masks, width = {}, {}
    for i in CBL_idx:
        # a BatchNorm-gamma threshold that keeps the chosen number of channels (obtain_bn_mask)
        root = find(i)
        if root not in width:
            width[root] = keep_width(name, defs, root, rs)
        gamma = loose.module_list[root][1].weight.data.abs()
        thre = torch.sort(gamma, descending=True)[0][min(width[root], gamma.numel()) - 1]
        masks[i] = pu.obtain_bn_mask(loose.module_list[root][1], thre).numpy()
    for i, d in enumerate(defs):     # depthwise / squeeze-excite layers keep their input's channels
        if d['type'] in ('depthwise', 'se'):
            masks[i] = pu.get_input_mask(defs, i, masks)
    compact_defs = deepcopy(defs)
    for i, mk in masks.items():
        compact_defs[i]['filters'] = str(int(mk.sum()))
    compact = ref_models.Darknet([loose.hyperparams.copy()] + compact_defs, img_size=(size, size))
    fresh = ref_models.Darknet([loose.hyperparams.copy()] + deepcopy(compact_defs), img_size=(size, size))
    pu.init_weights_from_loose_model(compact, loose, CBL_idx, Other_idx, masks)
    for i in Other_idx:
        t = defs[i]['type']
        if t not in ('depthwise', 'se'):
            continue
        keep = torch.from_numpy(np.argwhere(masks[i])[:, 0])
        cm, lm = compact.module_list[i], loose.module_list[i]
        if t == 'depthwise':
            cm[0].weight.data = lm[0].weight.data[keep].clone()
            for a in ('weight', 'bias', 'running_mean', 'running_var'):
                getattr(cm[1], a).data = getattr(lm[1], a).data[keep].clone()
        else:
            cr = fresh.module_list[i][0].fc[0].weight.shape[0]
            cm[0].fc[0].weight.data = lm[0].fc[0].weight.data[:cr][:, keep].clone()
            cm[0].fc[2].weight.data = lm[0].fc[2].weight.data[keep][:, :cr].clone()
    sd = compact.state_dict()
    bad = [(k, tuple(sd[k].shape), tuple(v.shape)) for k, v in fresh.state_dict().items() if sd[k].shape != v.shape]
    assert not bad, bad[:5]
    compact.eval()
    x = orc.synth_images(2, size, size, seed=5)
    with torch.no_grad():
        io = compact(x)[0]
    # the loose model is the stock cfg with synth_state_dict(seed 0): the fixture keeps the kept-channel indices and the
    # input-channel indices init_weights_from_loose_model used, not the weights, plus per-tensor sums to check a rebuild
    out = {"widths_json": np.array(json.dumps({str(i): int(mk.sum()) for i, mk in masks.items()})), "io": io.numpy(),
           "sd_names": np.array(sorted(sd)), "sd_sums": np.array([float(sd[k].double().sum()) for k in sorted(sd)])}
    for i, mk in masks.items():
        out["out%d" % i] = np.argwhere(mk)[:, 0].astype(np.int16)
    for i in CBL_idx + Other_idx:
        if defs[i]['type'] == 'convolutional':
            out["in%d" % i] = np.argwhere(pu.get_input_mask(defs, i, masks))[:, 0].astype(np.int16)
    widths = sorted({int(mk.sum()) for mk in masks.values()})
    print("%s %dpx: %d layers, widths %s" % (name, size, len(compact.module_defs), widths))
    return {"%s:%s" % (name, k): v for k, v in out.items()}


def main():
    out = {"cases": np.array(json.dumps([[n, s] for n, _, s in CASES]))}
    for name, cfg, size in CASES:
        out.update(build_case(name, cfg, size))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pruned_case.npz"), **out)


if __name__ == "__main__":
    main()
