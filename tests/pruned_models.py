"""The channel-pruned models of tests/golden/pruned_case.npz (oracle/gen_golden_pruned.py), rebuilt from the generated
stock cfgs: the loose model is the stock cfg with orc.synth_state_dict(seed 0); the fixture keeps the widths and the
kept output / input channels of every pruned layer."""
import json

import numpy as np
import torch

from helpers import cfg_path, golden, orc

_G = None


def fixture():
    global _G
    if _G is None:
        _G = golden("pruned_case")
    return _G


def cases():
    """[(name, image size)]"""
    return [tuple(c) for c in json.loads(str(fixture()["cases"]))]


def compact_defs(name):
    """parsed cfg ([net] first) with the pruned widths"""
    from utils.parse_config import parse_model_cfg
    defs = parse_model_cfg(cfg_path(name))
    for i, w in json.loads(str(fixture()[name + ":widths_json"])).items():
        defs[int(i) + 1]['filters'] = w
    return defs


def compact_state(name, template):
    """the loose model's synthetic parameters, cut down to the compact model's shapes the way
    init_weights_from_loose_model cuts them (depthwise and squeeze-excite layers keep their input's channels)"""
    import models
    g = fixture()
    loose = orc.synth_state_dict(models.Darknet(cfg_path(name)).state_dict(), 0)
    out = {}
    for k, v in template.items():
        i = int(k.split('.')[1])
        t = loose[k]
        o = torch.from_numpy(g["%s:out%d" % (name, i)].astype(np.int64)) if "%s:out%d" % (name, i) in g else None
        if '.se.fc.0.' in k:
            t = t[:v.shape[0]][:, o]
        elif '.se.fc.2.' in k:
            t = t[o][:, :v.shape[1]]
        elif t.dim() > 0:
            if o is not None:
                t = t[o]
            if t.dim() == 4 and "%s:in%d" % (name, i) in g:
                t = t[:, torch.from_numpy(g["%s:in%d" % (name, i)].astype(np.int64))]
        out[k] = t.clone()
    return out


def build_pruned(name, device=None):
    import models
    m = models.Darknet(compact_defs(name))
    m.load_state_dict(compact_state(name, m.state_dict()))
    return m.to(device) if device is not None else m


def images(name):
    size = dict(cases())[name]
    return orc.synth_images(2, size, size, seed=5)
