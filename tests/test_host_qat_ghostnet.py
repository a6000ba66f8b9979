"""CPU: the QAT module trees of yolov3-ghost.  Under google QAT (quantized=1) and TPSQ (quantized=2) every
[convolutional] block, GhostNet's depthwise cheap operations (groups=C) included, is one quantised BN-folded layer; the
fixtures (oracle/gen_golden_qat_ghostnet.py) record the reference's own trees and state_dict keys."""
import os
import tempfile

import pytest
import torch

from helpers import cfg_path, golden, orc

MODES = [(1, 1, "yolov3-ghost_64_qat1", "sw1."), (1, 2, "yolov3-ghost_64_qat1", "sw2."),
         (2, 1, "yolov3-ghost_64_qat2", "")]


def _qat(mode, shortcut_way=1):
    import models
    return models.Darknet(cfg_path("yolov3-ghost"), quantized=mode, a_bit=8, w_bit=8, shortcut_way=shortcut_way,
                          steps=100)


def _depthwise(m):
    return [b[0] for d, b in zip(m.module_defs, m.module_list) if d['type'] == 'convolutional' and b[0].groups != 1]


@pytest.mark.parametrize("mode,shortcut_way,fixture,prefix", MODES)
def test_ghost_qat_tree_and_keys_match_reference(mode, shortcut_way, fixture, prefix):
    g = golden(fixture)
    m = _qat(mode, shortcut_way)
    tree = ["%d %s %s" % (i, n, c.__class__.__name__) for i, b in enumerate(m.module_list) for n, c in b.named_children()]
    assert tree == [str(t) for t in g[prefix + "tree"]]
    ours, ref = list(m.state_dict().keys()), [str(k) for k in g[prefix + "state_keys"]]
    assert sorted(ours) == sorted(ref)
    # in order for the conv / se blocks (the quantised shortcuts register their trackers in another order)
    blocks = {str(i) for i, d in enumerate(m.module_defs) if d['type'] in ('convolutional', 'se')}
    assert [k for k in ours if k.split('.')[1] in blocks] == [k for k in ref if k.split('.')[1] in blocks]
    assert [n for n, _ in m.named_parameters()] == [str(k) for k in g[prefix + "param_names"]]
    dws = _depthwise(m)
    assert len(dws) == 41
    assert {(c.kernel_size[0], c.stride[0]) for c in dws} == {(3, 1), (3, 2), (5, 2)}
    for c in dws:
        assert c.groups == c.in_channels == c.out_channels and c.bias is None and c.bn
        assert hasattr(c, 'weight_quantizer') and c.weight.shape[1] == 1


@pytest.mark.parametrize("mode", [1, 2])
def test_ghost_qat_weights_round_trip(mode):
    """save_weights -> load_darknet_weights(quant=True): every slot back in place, the depthwise layers' [C, 1, k, k]
    weights and the BatchNorm held by each fold layer included"""
    import models
    m = _qat(mode)
    sd = orc.synth_state_dict(m.state_dict(), 3)
    m.load_state_dict({k: (sd[k] if v.is_floating_point() else v) for k, v in m.state_dict().items()})
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "q.weights")
        models.save_weights(m, path)
        m2 = _qat(mode)
        models.load_darknet_weights(m2, path, quant=True)
        slots = 0
        for mdef, b1, b2 in zip(m.module_defs, m.module_list, m2.module_list):
            for a, b in zip(models._weight_slots(mdef, b1, True), models._weight_slots(mdef, b2, True)):
                assert torch.equal(a, b)
                slots += a.numel()
        assert os.path.getsize(path) == 20 + 4 * slots
    for c1, c2 in zip(_depthwise(m), _depthwise(m2)):
        for name in ('beta', 'gamma', 'running_mean', 'running_var', 'weight'):
            assert torch.equal(getattr(c2, name), getattr(c1, name)), name


def test_google_grouped_convolution_raises():
    from utils.quantized.quantized_google import BNFold_QuantizedConv2d_For_FPGA
    c = BNFold_QuantizedConv2d_For_FPGA(16, 16, 3, padding=1, groups=4, bn=1, activate='relu', steps=100)
    with pytest.raises(NotImplementedError, match="grouped convolution"):
        c(torch.zeros(1, 8, 8, 16))


def test_ghost_keeps_the_qat_module_forwards_in_eval():
    from b200yolo.qengine import int8_graph_refusal
    assert int8_graph_refusal(_qat(1)) is not None
