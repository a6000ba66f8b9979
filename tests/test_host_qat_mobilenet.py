"""CPU: the google-QAT (quantized=1) module tree of yolov3-mobilenet.  The reference keeps its [depthwise] blocks in float
under quantized=1 (Conv2d(groups=C) + BatchNorm2d + activation) and its [se] layers as the float SE; the fixture
(oracle/gen_golden_qat_mobilenet.py) records the reference's own tree and state_dict keys."""
import os
import tempfile

import pytest
import torch

from helpers import cfg_path, golden, orc


def _qat(name, mode=1):
    import models
    return models.Darknet(cfg_path(name), quantized=mode, a_bit=8, w_bit=8, shortcut_way=1, steps=100)


def _tree(m):
    return ["%d %s %s" % (i, n, c.__class__.__name__) for i, b in enumerate(m.module_list) for n, c in b.named_children()]


def test_mobilenet_qat1_tree_and_keys_match_reference():
    g = golden("yolov3-mobilenet_64_qat1")
    m = _qat("yolov3-mobilenet")
    assert _tree(m) == [str(t) for t in g["tree"]]
    ours, ref = list(m.state_dict().keys()), [str(k) for k in g["state_keys"]]
    assert sorted(ours) == sorted(ref)
    # in order for the conv / depthwise / se blocks (the quantised shortcuts register their trackers in another order)
    blocks = {str(i) for i, d in enumerate(m.module_defs) if d['type'] in ('convolutional', 'depthwise', 'se')}
    assert [k for k in ours if k.split('.')[1] in blocks] == [k for k in ref if k.split('.')[1] in blocks]
    assert [n for n, _ in m.named_parameters()] == [str(k) for k in g["param_names"]]
    i = next(i for i, d in enumerate(m.module_defs) if d['type'] == 'depthwise')
    blk = m.module_list[i]
    assert isinstance(blk[0], torch.nn.Conv2d) and blk[0].groups == blk[0].in_channels and blk[0].bias is None
    assert isinstance(blk[1], torch.nn.BatchNorm2d) and blk[1].momentum == 0.1


def test_mobilenet_qat1_weights_round_trip():
    import models
    m = _qat("yolov3-mobilenet")
    sd = orc.synth_state_dict(m.state_dict(), 3)
    m.load_state_dict({k: (sd[k] if v.is_floating_point() else v) for k, v in m.state_dict().items()})
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "q.weights")
        models.save_weights(m, path)
        m2 = _qat("yolov3-mobilenet")
        models.load_darknet_weights(m2, path, quant=True)
        slots = 0
        for mdef, b1, b2 in zip(m.module_defs, m.module_list, m2.module_list):
            for a, b in zip(models._weight_slots(mdef, b1, True), models._weight_slots(mdef, b2, True)):
                assert torch.equal(a, b)
                slots += a.numel()
        assert os.path.getsize(path) == 20 + 4 * slots


@pytest.mark.parametrize("name", ["yolov3", "yolov3-tiny"])
@pytest.mark.parametrize("mode", [1, 2])
def test_yolov3_qat_trees_unchanged(name, mode):
    """no [depthwise] block in these cfgs: every conv stays a single quantised module"""
    m = _qat(name, mode)
    for d, b in zip(m.module_defs, m.module_list):
        if d['type'] == 'convolutional':
            assert [n for n, _ in b.named_children()] == ['Conv2d']
            assert hasattr(b[0], 'weight_quantizer')


def test_mobilenet_tpsq_keeps_quantised_depthwise():
    m = _qat("yolov3-mobilenet", 2)
    i = next(i for i, d in enumerate(m.module_defs) if d['type'] == 'depthwise')
    assert [n for n, _ in m.module_list[i].named_children()] == ['DepthWise2d']
    assert hasattr(m.module_list[i][0], 'weight_quantizer')
