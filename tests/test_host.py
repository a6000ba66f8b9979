"""CPU: host-side logic -- cfg parser, generated cfgs, Darknet module tree / state_dict contract, .weights IO known
answers, C-ABI export check (no compute: there is no GPU here)."""
import ctypes
import json
import os
import re
import tempfile

import numpy as np
import pytest
import torch

from helpers import GOLD, PKG, ROOT, cfg_path, module_defs, orc, stem_model

def _snapshot():
    with open(os.path.join(GOLD, "cfg_snapshot.json")) as f:
        return json.load(f)


def test_c_abi_exports_every_declared_symbol():
    """every function declared in include/b200yolo.h is exported by libb200yolo.so and bound in b200yolo.lib."""
    with open(os.path.join(ROOT, "include", "b200yolo.h")) as f:
        hdr = f.read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = sorted(set(re.findall(r"\b(b2y_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) > 40
    so = os.path.join(PKG, "libb200yolo.so")
    assert os.path.exists(so), "run python __graft_entry__.py (build) first"
    lib = ctypes.CDLL(so)
    missing = [n for n in declared if not hasattr(lib, n)]
    assert not missing, missing
    from b200yolo import lib as binding
    assert not binding.MISSING
    unbound = [n for n in declared if n not in binding.EXPORTS and n != "b2y_set_last_cuda_error"]
    assert not unbound, "declared in the header but not bound in b200yolo/lib.py: %s" % unbound
    assert lib.b2y_abi_version() == 3
    assert binding.raw().b2y_strerror(-3).decode().startswith("unsupported")


def test_parser_rules():
    from utils.parse_config import parse_model_cfg_text
    text = """[net]
width=416
momentum=0.949
# comment
[convolutional]
filters=32
size=3
stride=1
pad=1
activation=leaky

[depthwise]
filters=32
size=3,5
stride=1
pad=1
activation=linear
[yolo]
mask = 0,1
anchors = 10,14,  23,27
classes=2
num=2
jitter=.3
scale_x_y = 1.05
"""
    d = parse_model_cfg_text(text)
    assert d[0]['type'] == 'net' and d[0]['width'] == 416 and d[0]['momentum'] == '0.949'
    assert d[1]['batch_normalize'] == 0 and d[1]['filters'] == 32 and d[1]['activation'] == 'leaky'
    assert 'batch_normalize' not in d[2] and d[2]['size'] == [3, 5]
    assert d[3]['mask'] == [0, 1] and d[3]['anchors'].shape == (2, 2) and d[3]['anchors'].dtype == np.float64
    assert d[3]['jitter'] == '.3' and d[3]['scale_x_y'] == '1.05' and d[3]['classes'] == 2
    with pytest.raises(AssertionError):
        parse_model_cfg_text("[net]\n[convolutional]\nbogus_key=1\n")


@pytest.mark.parametrize("name", ["yolov3-tiny", "yolov3", "yolov4"])
def test_model_tree_matches_reference_snapshot(name):
    import models
    snap = _snapshot()[name]
    m = models.Darknet(cfg_path(name))
    assert len(m.module_list) == snap["modules"]
    assert sum(1 for d in m.module_defs if d['type'] == 'convolutional') == snap["convs"]
    assert sum(p.numel() for p in m.parameters()) == snap["params"]
    assert list(m.yolo_layers) == snap["yolo_layers"]
    assert [int(m.module_list[j].stride) for j in m.yolo_layers] == snap["strides"]
    keys = list(m.state_dict().keys())
    assert keys[:8] == snap["state_keys_head"] and len(keys) == snap["n_state_keys"]
    # .weights: byte-exact size (== official darknet files) and bit-exact round trip
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "w.weights")
        m.load_state_dict(orc.synth_state_dict(m.state_dict(), 0))
        models.save_weights(m, path)
        assert os.path.getsize(path) == snap["weights_bytes"]
        m2 = models.Darknet(cfg_path(name))
        models.load_darknet_weights(m2, path)
        for (k, a), (_, b) in zip(m.state_dict().items(), m2.state_dict().items()):
            if not k.endswith("num_batches_tracked"):
                assert torch.equal(a, b), k
        with open(path, "rb") as f:
            assert np.frombuffer(f.read(12), dtype=np.int32).tolist() == [0, 2, 5]
        with open(path, "ab") as f:  # trailing garbage -> the loader's length assert fires (models.py:735)
            f.write(b"\0\0\0\0")
        with pytest.raises(AssertionError):
            models.load_darknet_weights(m2, path)


def test_module_layout_contract():
    """what the reference's scripts reach into: module_list[i][0]/[1], names, optimiser grouping substrings."""
    import models
    import torch.nn as nn
    m = models.Darknet(cfg_path("yolov3-tiny"), FPGA=False)   # detect.py:26 passes FPGA=
    blk = m.module_list[0]
    assert [n for n, _ in blk.named_children()] == ['Conv2d', 'BatchNorm2d', 'activation']
    assert isinstance(blk[0], nn.Conv2d) and isinstance(blk[1], nn.BatchNorm2d) and blk[1].momentum == 0.1
    assert isinstance(blk[2], nn.LeakyReLU) and blk[2].negative_slope == 0.1
    names = dict(m.named_parameters())
    assert 'module_list.0.Conv2d.weight' in names and 'module_list.0.BatchNorm2d.bias' in names
    assert m.module_list[16].__class__.__name__ == 'YOLOLayer' and m.module_list[17].__class__.__name__ == 'FeatureConcat'
    y = m.module_list[16]
    assert y.na == 3 and y.no == 85 and y.anchor_vec.shape == (3, 2)
    assert torch.allclose(y.anchor_vec, y.anchors / y.stride)
    assert m.module_defs[0]['type'] == 'convolutional' and m.hyperparams['type'] == 'net'
    head = m.module_list[15][0]   # smart bias init (models.py:325-335)
    assert torch.allclose(head.bias.view(3, -1)[:, 4].mean(), torch.tensor(-4.5), atol=0.2)
    # cfg passed as a list of defs (pruning scripts)
    from utils.parse_config import parse_model_cfg
    m2 = models.Darknet(parse_model_cfg(cfg_path("yolov3-tiny")))
    assert len(m2.module_list) == 24
    import copy
    m3 = copy.deepcopy(m)     # ModelEMA deep-copies the model
    assert len(m3.module_list) == 24 and m3._engine is None


def test_fuse_matches_oracle_fold():
    import models
    m = models.Darknet(cfg_path("yolov3-tiny"))
    m.load_state_dict(orc.synth_state_dict(m.state_dict(), 0))
    sd = m.state_dict()
    w, b = orc.fold_bn(sd['module_list.2.Conv2d.weight'], None, sd['module_list.2.BatchNorm2d.weight'],
                       sd['module_list.2.BatchNorm2d.bias'], sd['module_list.2.BatchNorm2d.running_mean'],
                       sd['module_list.2.BatchNorm2d.running_var'], 1e-5)
    m.fuse()
    fused = m.module_list[2][0]
    assert [n for n, _ in m.module_list[2].named_children()] == ['0', '1']
    assert torch.allclose(fused.weight, w, rtol=1e-5, atol=1e-7) and torch.allclose(fused.bias, b, rtol=1e-5, atol=1e-6)


def test_cpu_tensors_fail_loudly():
    import models
    m = models.Darknet(cfg_path("yolov3-tiny")).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 64, 64))
    from utils import utils as my_utils
    with pytest.raises(RuntimeError, match="CUDA"):
        my_utils.compute_loss([torch.zeros(1, 3, 2, 2, 85)], torch.zeros(0, 6), m)


_LAYOUT_CFG = """
[net]
width=96
height=96
channels=3
""" + "".join("\n[%s]\n%s\n" % (kind, "\n".join(opts.split())) for kind, opts in (
    ("convolutional", "batch_normalize=1 filters=16 size=3 stride=1 pad=1 activation=leaky"),     # 0
    ("convolutional", "batch_normalize=1 filters=32 size=3 stride=2 pad=1 activation=leaky"),     # 1
    ("route", "layers=-1 groups=2 group_id=1"),                                                   # 2 upper half of 1
    ("convolutional", "batch_normalize=1 filters=16 size=3 stride=1 pad=1 activation=leaky"),     # 3
    ("convolutional", "batch_normalize=1 filters=16 size=3 stride=1 pad=1 activation=leaky"),     # 4
    ("route", "layers=-1,-2"),                                                                    # 5
    ("convolutional", "batch_normalize=1 filters=32 size=1 stride=1 pad=1 activation=leaky"),     # 6
    ("route", "layers=-6,-1"),                                                                    # 7 = [1 | 6]
    ("maxpool", "size=2 stride=2"),                                                               # 8
    ("convolutional", "batch_normalize=1 filters=32 size=1 stride=1 pad=1 activation=leaky"),     # 9
    ("convolutional", "batch_normalize=1 filters=64 size=3 stride=1 pad=1 activation=leaky"),     # 10
    ("shortcut", "from=-2 activation=linear"),                                                    # 11 addend narrower
    ("route", "layers=-1"),                                                                       # 12 = 11
    ("route", "layers=-1"),                                                                       # 13 = 12 = 11
    ("convolutional", "batch_normalize=1 filters=32 size=1 stride=1 pad=1 activation=leaky"),     # 14
    ("route", "layers=-1,-3"),                                                                    # 15 = [14 | 11]
    ("convolutional", "batch_normalize=1 filters=32 size=1 stride=1 pad=1 activation=leaky"),     # 16
    ("route", "layers=-1,11"),                                                                    # 17: 11 is taken
    ("convolutional", "batch_normalize=1 filters=64 size=3 stride=1 pad=1 activation=leaky"),     # 18
    ("convolutional", "batch_normalize=1 filters=64 size=1 stride=1 pad=1 activation=leaky"),     # 19
    ("convolutional", "batch_normalize=1 filters=64 size=3 stride=1 pad=1 activation=leaky"),     # 20
    ("shortcut", "from=-3 activation=linear"),                                                    # 21 into conv 20
    ("convolutional", "filters=64 size=1 stride=1 pad=1 activation=linear"),                      # 22 no BatchNorm
    ("shortcut", "from=-2 activation=linear"),                                                    # 23
    ("convolutional", "filters=255 size=1 stride=1 pad=1 activation=linear"),                     # 24
    ("yolo", "mask=0,1,2 anchors=10,14,23,27,37,58,81,82,135,169,344,319 classes=80 num=6")))     # 25


def test_layout_is_decided_once_for_inference_and_training():
    """b200yolo.layout on the CPU: shapes, folded shortcuts per mode, aliases, zero-copy concat placement."""
    import models
    from b200yolo import layout
    from utils.parse_config import parse_model_cfg_text

    def layouts(model, chw=(3, 96, 160)):
        shapes = layout.infer_shapes(model, chw)
        bn_of = lambda i: layout._block_parts(model.module_list[i])[1]
        return (layout.build_layout(model, shapes, False, lambda i: shapes[i][0] % 8 == 0),
                layout.build_layout(model, shapes, False, lambda i: bn_of(i) is not None),
                layout.build_layout(model, shapes, True, lambda i: True))
    n_fused = lambda lay: sum(f is not None for f in lay.fused_into)

    # shortcuts folded into the conv before them (inference, training, keep_features), feature_out entries
    for name, want in (("yolov3", (23, 23, 0, 72)), ("yolov3-tiny", (0, 0, 0, 12)), ("yolov4", (23, 23, 0, 107)),
                       ("yolov3-mobilenet", (10, 10, 0, 75))):
        model = models.Darknet(cfg_path(name))
        inf, trn, keep = layouts(model)
        assert (n_fused(inf), n_fused(trn), n_fused(keep), len(layout.feature_slots(model))) == want, name
        if name == "yolov4":    # every concat source is written in place, SPP included
            assert sorted(inf.concats) == [9, 22, 53, 84, 103, 113, 121, 131, 142, 153]
            assert all(placed for parts in inf.concats.values() for _, _, placed in parts)
            assert [off for _, off, _ in inf.concats[113]] == [0, 512, 1024, 1536]
            assert inf.shapes[113] == (2048, 3, 5)
        if name == "yolov3-tiny":   # the 2/1 max-pool keeps the size
            assert inf.shapes[10] == inf.shapes[11] == (512, 3, 5)
        if name == "yolov3-mobilenet":
            odd = sorted({(t.C, layout.pitch(t.C, t.dtype)) for t in inf.tens if t is not None and t.C % 16})
            assert odd == [(24, 32), (40, 48), (72, 80), (120, 128), (168, 176), (184, 192), (200, 208), (255, 256)]

    model = models.Darknet(parse_model_cfg_text(_LAYOUT_CFG))
    inf, trn, keep = layouts(model)
    assert (n_fused(inf), n_fused(trn), n_fused(keep)) == (2, 1, 0)     # conv 22 has no BatchNorm
    assert inf.fused_into[21] == trn.fused_into[21] == 20 and inf.fused_into[11] is None
    assert inf.fused_into[23] == 22 and trn.fused_into[23] is None
    for lay in (inf, trn):
        t = lay.tens
        assert lay.shapes[2] == (16, 48, 80) and lay.shapes[8] == (64, 24, 40) and lay.shapes[17] == (96, 24, 40)
        assert t[12] is t[11] and t[13] is t[11] and t[20] is t[21] and t[25] is None
        # conv 1 sits at the start of concat 7; the grouped route is the upper half of its channels, same buffer
        assert lay.concats[7] == [(t[1], 0, True), (t[6], 32, True)]
        assert lay.grouped == {2: t[1]} and (t[2].c0, t[2].C) == (t[1].c0 + 16, 16)
        assert lay.concats[5] == [(t[4], 0, True), (t[3], 16, True)]
        assert lay.concats[15] == [(t[14], 0, True), (t[11], 32, True)]
        assert lay.concats[17] == [(t[16], 0, True), (t[11], 32, False)]     # already inside concat 15: copied
        assert t[11].c0 == 32 and t[24].dtype == torch.float32 and lay.is_head[24]

    model = models.Darknet(parse_model_cfg_text(_LAYOUT_CFG.replace("[maxpool]", "[reorg3d]")))
    with pytest.raises(NotImplementedError, match="reorg3d"):
        layout.infer_shapes(model, (3, 96, 96))
    with pytest.raises(NotImplementedError, match="int8 graph"):
        layout.infer_shapes(models.Darknet(cfg_path("yolov3-tiny")), (3, 96, 96), ('convolutional', 'yolo'),
                            "layer type '%s' in the int8 graph")


def test_stem_path_follows_the_compiled_shape_list():
    """layout.stem_path picks an im2col kernel only for an (in_c, k) pair that csrc/common.cuh compiles them for, and
    the training plans record its choice; the gradient plan refuses, naming the layer, every first layer whose direct
    weight gradient b2y_stem_conv_bwd_weight cannot take (more than 40 taps)."""
    from b200yolo import layout
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainPlan, TrainShared
    with open(os.path.join(PKG, "csrc", "common.cuh")) as f:
        line = re.search(r"#define B2Y_STEM_IM2COL_SHAPES\(X\)(.*)", f.read()).group(1)
    listed = {(int(c), int(k)) for c, k in re.findall(r"X\((\d+), (\d+)\)", line)}
    assert (3, 3) in listed and (1, 3) in listed
    dev = torch.device("cpu")
    for in_c in range(1, 5):
        for k in range(1, 8):
            on_list = (in_c, k) in listed
            for out_c in (16, 32, 64, 72, 256):
                want = ('fused' if out_c <= 64 else 'im2col') if on_list else 'direct'
                assert layout.stem_path(in_c, k, out_c) == want, (in_c, k, out_c)
                assert layout.stem_path(in_c, k, out_c, training=True) == ('im2col' if on_list else 'direct')
                assert layout.stem_path(in_c, k, out_c, training=True, batch_norm=False) == 'direct'
            for stride in (1, 2):
                model = stem_model(in_c, k, stride).train()
                shape = (2, in_c, 40, 48)
                fo = TrainPlan(model, shape, dev, False, SlotStore(dev), TrainShared(dev), forward_only=True)
                assert fo.convs[0].stem == ('im2col' if on_list else 'direct')
                if fo.convs[0].stem == 'direct' and in_c * k * k > layout.STEM_WGRAD_MAX_TAPS:
                    with pytest.raises(NotImplementedError, match="layer 0: the weight gradient of a %dx%d first "
                                                                  "layer on %d channels" % (k, k, in_c)):
                        TrainPlan(model, shape, dev, False, SlotStore(dev), TrainShared(dev))
                else:
                    plan = TrainPlan(model, shape, dev, False, SlotStore(dev), TrainShared(dev))
                    assert plan.convs[0].stem == fo.convs[0].stem
    with pytest.raises(NotImplementedError, match="more than 4 input channels"):
        layout.stem_path(5, 3, 32)


@pytest.mark.parametrize("name", ["yolov3", "yolov3-tiny", "yolov4", "yolov3-mobilenet"])
def test_generated_cfg_equals_reference_cfg(name):
    """the generated cfgs against the reference's own .cfg files, as parsed (tests/golden/ref_cfg_layers.json,
    written by oracle/gen_golden_cfg.py)."""
    with open(os.path.join(GOLD, "ref_cfg_layers.json")) as f:
        ref = json.load(f)[name]
    ours = module_defs(name)
    assert len(ours) == len(ref)
    keys = ('type', 'batch_normalize', 'filters', 'size', 'stride', 'pad', 'activation', 'layers', 'from', 'mask',
            'classes', 'num')

    def plain(v):
        return v.tolist() if hasattr(v, "tolist") else v
    for a, b in zip(ours, ref):
        for k in keys:
            assert plain(a.get(k)) == b.get(k), (name, k, a, b)
        if 'anchors' in b:
            assert np.array_equal(np.asarray(a['anchors']), np.asarray(b['anchors']))


def test_prepare_labels_matches_the_reference_expressions():
    """b200yolo.detect.prepare_labels (host-side torch ops feeding the TP-matching kernel) against test.py:124, 145-148
    evaluated image by image: labels = targets[targets[:, 0] == si, 1:]; tbox = xywh2xyxy(labels[:, 1:5]) * whwh."""
    import torch
    from b200yolo import detect
    from utils import utils as U
    g = torch.Generator().manual_seed(4)
    B, W, H = 5, 640, 416
    t = torch.rand(23, 6, generator=g)
    t[:, 0] = torch.tensor([3, 0, 0, 4, 3, 1, 0, 4, 4, 1, 3, 0, 1, 1, 0, 3, 4, 0, 1, 3, 0, 4, 1]).float()   # image 2 is empty
    t[:, 1] = torch.randint(0, 80, (23,), generator=g).float()
    tcls, tbox, lab_off = detect.prepare_labels(t, B, W, H, torch.device("cpu"))
    whwh = torch.tensor([W, H, W, H], dtype=torch.float32)
    off = 0
    for si in range(B):
        labels = t[t[:, 0] == si, 1:]
        n = labels.shape[0]
        assert int(lab_off[si]) == off and int(lab_off[si + 1]) == off + n
        if n:
            assert torch.equal(tcls[off:off + n], labels[:, 0])
            assert torch.equal(tbox[off:off + n], U.xywh2xyxy(labels[:, 1:5]) * whwh)
        off += n
    e = detect.prepare_labels(torch.zeros(0, 6), B, W, H, torch.device("cpu"))
    assert e[0].numel() == 0 and e[1].shape == (0, 4) and e[2].tolist() == [0] * (B + 1)
