"""CPU: the TPSQ (quantized=2) module tree of yolov3-mobilenet.  Every [depthwise] block is one quantised, BN-folded
TPSQ_BNFold_QuantizedConv2d_For_FPGA(groups=C) named DepthWise2d; the fixture (oracle/gen_golden_qat2_mobilenet.py)
records the reference's own tree and state_dict keys."""
import os
import tempfile

import pytest
import torch

from helpers import cfg_path, golden, orc


def _tpsq(name="yolov3-mobilenet"):
    import models
    return models.Darknet(cfg_path(name), quantized=2, a_bit=8, w_bit=8, shortcut_way=1, steps=100)


def test_mobilenet_tpsq_tree_and_keys_match_reference():
    g = golden("yolov3-mobilenet_64_qat2")
    m = _tpsq()
    tree = ["%d %s %s" % (i, n, c.__class__.__name__) for i, b in enumerate(m.module_list) for n, c in b.named_children()]
    assert tree == [str(t) for t in g["tree"]]
    ours, ref = list(m.state_dict().keys()), [str(k) for k in g["state_keys"]]
    assert sorted(ours) == sorted(ref)
    blocks = {str(i) for i, d in enumerate(m.module_defs) if d['type'] in ('convolutional', 'depthwise', 'se')}
    assert [k for k in ours if k.split('.')[1] in blocks] == [k for k in ref if k.split('.')[1] in blocks]
    assert [n for n, _ in m.named_parameters()] == [str(k) for k in g["param_names"]]
    dws = [m.module_list[i][0] for i, d in enumerate(m.module_defs) if d['type'] == 'depthwise']
    assert len(dws) == 15
    for c in dws:
        assert c.groups == c.in_channels == c.out_channels and c.bias is None and c.bn and c.momentum == 0.01


def test_tpsq_grouped_convolution_raises():
    from utils.quantized.quantized_TPSQ import TPSQ_BNFold_QuantizedConv2d_For_FPGA
    c = TPSQ_BNFold_QuantizedConv2d_For_FPGA(16, 16, 3, padding=1, groups=4, bn=1, activate='relu6', steps=100)
    with pytest.raises(NotImplementedError, match="grouped convolution"):
        c(torch.zeros(1, 8, 8, 16))


def test_mobilenet_tpsq_weights_round_trip_keeps_depthwise_bn_in_place():
    """save_weights -> load_darknet_weights(quant=True) puts every depthwise layer's beta, gamma and running statistics
    back into that layer (the reference's own loader writes them into the preceding [convolutional] module)."""
    import models
    m = _tpsq()
    sd = orc.synth_state_dict(m.state_dict(), 3)
    m.load_state_dict({k: (sd[k] if v.is_floating_point() else v) for k, v in m.state_dict().items()})
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "q.weights")
        models.save_weights(m, path)
        m2 = _tpsq()
        models.load_darknet_weights(m2, path, quant=True)
    n = 0
    for mdef, b1, b2 in zip(m.module_defs, m.module_list, m2.module_list):
        for a, b in zip(models._weight_slots(mdef, b1, True), models._weight_slots(mdef, b2, True)):
            assert torch.equal(a, b)
        if mdef['type'] == 'depthwise':
            for name in ('beta', 'gamma', 'running_mean', 'running_var', 'weight'):
                assert torch.equal(getattr(b2[0], name), getattr(b1[0], name)), name
            n += 1
    assert n == 15
