"""Shared test helpers: golden loader, generated cfgs, model + oracle construction with identical synthetic weights."""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PKG = os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200")
GOLD = os.path.join(HERE, "golden")
for p in (PKG, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import darknet_oracle as orc  # noqa: E402

_CFG_DIR = None


def cfg_path(name):
    """Write the generated cfg once per session; the file name keeps e.g. 'yolov4' (stride order keys on it)."""
    global _CFG_DIR
    from b200yolo import cfggen
    if _CFG_DIR is None:
        _CFG_DIR = tempfile.mkdtemp(prefix="b2y_cfg_")
    path = os.path.join(_CFG_DIR, name + ".cfg")
    if not os.path.exists(path):
        cfggen.write_cfg(name, _CFG_DIR)
    return path


def module_defs(name):
    from utils.parse_config import parse_model_cfg
    return parse_model_cfg(cfg_path(name))[1:]


def golden(name):
    return np.load(os.path.join(GOLD, name + ".npz"), allow_pickle=False)


def build_model(name, seed=0, device=None):
    """Our Darknet with the deterministic synthetic parameters of oracle.synth_state_dict."""
    import models
    m = models.Darknet(cfg_path(name))
    m.load_state_dict(orc.synth_state_dict(m.state_dict(), seed))
    if device is not None:
        m = m.to(device)
    return m


def attach_hyp(m, nc=80):
    m.nc, m.hyp, m.gr = nc, dict(orc.DEFAULT_HYP), 1.0
    m.hyp['cls'] = m.hyp['cls'] * nc / 80.0
    return m


def anchor_vecs(name):
    defs = module_defs(name)
    ys = [d for d in defs if d['type'] == 'yolo']
    strides = orc.yolo_strides(name, len(ys))
    return [torch.as_tensor(np.asarray(d['anchors'])[d['mask']], dtype=torch.float32) / s for d, s in zip(ys, strides)]


STEM_CFG = """[net]
width=64
height=64
channels=3

[convolutional]
batch_normalize=1
filters=%d
size=%d
stride=%d
pad=1
activation=leaky

[convolutional]
size=1
stride=1
pad=1
filters=18
activation=linear

[yolo]
mask=0,1,2
anchors=10,14,23,27,37,58
classes=1
num=3
"""


def stem_model(in_c, k, stride, filters=32, seed=0, device=None):
    """A first-layer conv (k x k, stride, BatchNorm, leaky) on in_c input channels and a one-class YOLO head behind a
    1x1 conv, with the synthetic parameters of oracle.synth_state_dict.  The cfg format fixes 3 input channels, so the
    first conv is replaced by one on in_c."""
    import models
    from utils.parse_config import parse_model_cfg_text
    m = models.Darknet(parse_model_cfg_text(STEM_CFG % (filters, k, stride)))
    m.module_list[0].Conv2d = torch.nn.Conv2d(in_c, filters, k, stride, (k - 1) // 2, bias=False)
    m.load_state_dict(orc.synth_state_dict(m.state_dict(), seed))
    return m if device is None else m.to(device)
