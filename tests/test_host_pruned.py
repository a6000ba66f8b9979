"""CPU: channel-pruned models in the layer layout (logical width C stored as Cp = whole 8-channel groups), the weight
scatter that gives pad and gap channels zero weights, and the oracle against the reference's outputs on the pruned
fixture models (tests/golden/pruned_case.npz, oracle/gen_golden_pruned.py)."""
import pytest
import torch
import torch.nn.functional as F

from helpers import cfg_path, orc
from pruned_models import build_pruned, cases, compact_defs, fixture, images

CASES = [n for n, _ in cases()]


def _plan(model, S, keep):
    from b200yolo import engine
    return engine.Plan(model, (2, 3, S, S), torch.device("cpu"), keep)


def _layout(model, S):
    from b200yolo import layout
    shapes = layout.infer_shapes(model, (3, S, S))
    return layout.build_layout(model, shapes, False, lambda i: True)


@pytest.mark.parametrize("name", ["yolov3", "yolov3-tiny", "yolov4", "yolov3-mobilenet"])
def test_stock_cfgs_keep_their_layout(name):
    """every stock width is a multiple of 8: physical = logical everywhere, so the plans are the ones before"""
    import models
    from b200yolo import cfggen, layout
    assert name in cfggen.ARCHS
    model = models.Darknet(cfg_path(name))
    for keep in (False, True):
        plan = _plan(model, 96, keep)
        lay = _layout(model, 96)
        for i, t in enumerate(lay.tens):
            if t is None:
                continue
            assert t.Cp == t.C and lay.chmap[i] == tuple(range(t.C)), (name, i)
        for i, parts in lay.concats.items():
            offs = [off for _, off, _ in parts]
            assert offs == [sum(st.C for st, _, _ in parts[:j]) for j in range(len(parts))]
        for st in plan.steps:
            for f in st:
                if isinstance(f, layout._Tensor) and f.dtype == torch.float16:
                    assert f.view().shape[3] == f.C


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("keep", [False, True])
def test_pruned_layout_is_in_whole_8_channel_groups(name, keep):
    from b200yolo import layout
    model = build_pruned(name)
    S = dict(cases())[name]
    plan = _plan(model, S, keep)
    lay = _layout(model, S)
    assert any(t is not None and t.C % 8 for t in lay.tens), "the fixture has pruned widths"
    for i, t in enumerate(lay.tens):
        if t is None:
            continue
        m = lay.chmap[i]
        assert len(m) == t.C and all(a < b for a, b in zip(m, m[1:])) and m[-1] < t.Cp, (name, i)
        if t.dtype == torch.float16:
            assert t.Cp % 8 == 0, (name, i)
        else:
            assert lay.is_head[i] and t.Cp == t.C
    gapped = 0
    for i, parts in lay.concats.items():
        off, want = 0, ()
        for (st, o, placed), s in zip(parts, layout.sources(i, model.module_defs[i]['layers'])):
            assert o == off and o % 8 == 0 and lay.tens[s] is st
            if placed:
                assert st.c0 == o
            want += tuple(o + c for c in lay.chmap[s])
            off += st.Cp
        assert lay.tens[i].Cp == off and lay.chmap[i] == want
        gapped += lay.chmap[i] != tuple(range(lay.tens[i].C))
    if name == "yolov3-tiny":
        # route 20 = [upsample of conv 18 (37 channels) | conv 8 (37 channels)]: the second source sits at channel 40
        assert [(o, st.C, st.Cp) for st, o, _ in lay.concats[20]] == [(0, 37, 40), (40, 37, 40)]
        assert lay.chmap[20] == tuple(range(37)) + tuple(range(40, 77))
        assert gapped
    # every kernel launch sees whole 8-channel groups; a conv's padded K view stays inside its source's buffer
    for st in plan.steps:
        if st.kind == 'conv' and st.src is not None:
            assert st.src.view_k().shape[3] % 16 == 0
        for f in st:
            if isinstance(f, layout._Tensor) and f.dtype == torch.float16:
                v = f.view()
                assert v.shape[3] % 8 == 0 and (f.c0 % 8 == 0) and f.c0 + f.Cp <= f.buf.shape[3]


def test_weight_scatter_matches_the_compact_conv():
    """the padded weight on a zero-gapped input equals the compact conv on the compact input (fp32), and the pad outputs
    are exactly zero; the same for the depthwise fold"""
    from b200yolo import engine
    model = build_pruned("yolov3-tiny")
    lay = _layout(model, 96)
    g = torch.Generator().manual_seed(0)
    for i in (21, 14):            # reads the gapped concat [37 | 37]; reads a 100-channel (= 4 mod 8) tensor
        conv = model.module_list[i][0]
        src, out = lay.tens[i - 1], lay.tens[i]
        K = (src.Cp + 15) // 16 * 16
        w = conv.weight.detach()
        b = torch.randn(conv.out_channels, generator=g)
        wp = engine._scatter(engine._pad_rows(w, out.Cp), 1, lay.chmap[i - 1], K)
        bp = engine._pad_rows(b, out.Cp)
        x = torch.randn(2, src.C, 13, 11, generator=g)
        xg = torch.zeros(2, K, 13, 11)
        xg[:, list(lay.chmap[i - 1])] = x
        p = conv.padding[0]
        y = F.conv2d(x.double(), w.double(), b.double(), padding=p)
        yp = F.conv2d(xg.double(), wp.double(), bp.double(), padding=p)
        assert out.Cp > out.C or src.Cp > src.C
        assert torch.equal(yp[:, out.C:], torch.zeros_like(yp[:, out.C:]))
        assert ((yp[:, :out.C] - y).abs().max() / y.abs().max()).item() < 1e-6
        y32 = F.conv2d(xg, wp, bp, padding=p)[:, :out.C]
        assert ((y32 - y.float()).abs().max() / y.abs().max()).item() < 1e-6
    # depthwise: pad channels get zero weights, scale and bias
    mob = build_pruned("yolov3-mobilenet")
    lay = _layout(mob, 128)
    i = next(i for i, d in enumerate(mob.module_defs) if d['type'] == 'depthwise' and lay.tens[i].Cp > lay.tens[i].C)
    conv, bn = mob.module_list[i][0], mob.module_list[i][1]
    cmap, cp = lay.chmap[i - 1], lay.tens[i - 1].Cp
    sc, bi = engine.fold_bn(conv, bn)
    wp, scp, bip = (engine._scatter(t, 0, cmap, cp) for t in (conv.weight.detach(), sc, bi))
    C = conv.in_channels
    x = torch.randn(2, C, 9, 9, generator=g)
    xg = torch.zeros(2, cp, 9, 9)
    xg[:, list(cmap)] = x
    k = conv.kernel_size[0]
    y = F.conv2d(x, conv.weight.detach(), None, conv.stride, conv.padding, 1, C) * sc.view(1, -1, 1, 1) + bi.view(1, -1, 1, 1)
    yp = F.conv2d(xg, wp, None, conv.stride, conv.padding, 1, cp) * scp.view(1, -1, 1, 1) + bip.view(1, -1, 1, 1)
    assert k in (3, 5) and torch.equal(yp[:, C:], torch.zeros_like(yp[:, C:]))
    assert ((yp[:, list(cmap)] - y).abs().max() / y.abs().max()).item() < 1e-6


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_on_pruned_models(name):
    import numpy as np
    g = fixture()
    model = build_pruned(name)
    sd = model.state_dict()
    names = sorted(sd)
    assert names == [str(s) for s in g[name + ":sd_names"]]
    # the rebuilt compact parameters are the ones the reference's init_weights_from_loose_model produced
    np.testing.assert_array_equal([float(sd[k].double().sum()) for k in names], g[name + ":sd_sums"])
    with torch.no_grad():
        io, _ = orc.darknet_forward(compact_defs(name)[1:], sd, images(name), name)
    ref = torch.from_numpy(g[name + ":io"])
    assert io.shape == ref.shape
    box = ((io[..., :4] - ref[..., :4]).abs() / ref[..., :4].abs().clamp(min=1.0)).max().item()
    prob = (io[..., 4:] - ref[..., 4:]).abs().max().item()
    assert box < 1e-5 and prob < 1e-5, (box, prob)


def test_training_plan_refuses_pruned_widths():
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainPlan, TrainShared
    dev = torch.device("cpu")
    for name, S in cases():
        with pytest.raises(NotImplementedError, match=r"layer \d+: BatchNorm training needs a multiple of 8"):
            TrainPlan(build_pruned(name), (2, 3, S, S), dev, False, SlotStore(dev), TrainShared(dev))


_CFG = """
[net]
width=96
height=96
channels=3
""" + "".join("\n[%s]\n%s\n" % (kind, "\n".join(opts.split())) for kind, opts in (
    ("convolutional", "batch_normalize=1 filters=16 size=3 stride=1 pad=1 activation=leaky"),     # 0
    ("convolutional", "batch_normalize=1 filters=%d size=3 stride=2 pad=1 activation=leaky"),     # 1
    ("route", "layers=-1 groups=2 group_id=1"),                                                   # 2 upper half of 1
    ("convolutional", "batch_normalize=1 filters=%d size=3 stride=1 pad=1 activation=leaky"),     # 3
    ("shortcut", "from=-3 activation=linear"),                                                    # 4
    ("convolutional", "filters=255 size=1 stride=1 pad=1 activation=linear"),                     # 5
    ("yolo", "mask=0,1,2 anchors=10,14,23,27,37,58,81,82,135,169,344,319 classes=80 num=6")))     # 6


def test_unsupported_pruned_routes_and_shortcuts_fail_at_plan_build():
    import models
    from utils.parse_config import parse_model_cfg_text
    # 48 channels: the upper half starts at channel 24, a whole 8-channel group
    lay = _layout(models.Darknet(parse_model_cfg_text(_CFG % (48, 24))), 96)
    assert (lay.tens[2].c0, lay.tens[2].C, lay.tens[2].Cp) == (24, 24, 24)
    for w in (40, 37):
        with pytest.raises(NotImplementedError, match="layer 2: grouped route"):
            _layout(models.Darknet(parse_model_cfg_text(_CFG % (w, 24))), 96)
    # 20-channel conv 3 plus the 48-channel conv 1: the sum would spill conv 1's channels 20..23 into the pad
    with pytest.raises(NotImplementedError, match="layer 4: shortcut whose addend is wider"):
        _layout(models.Darknet(parse_model_cfg_text(_CFG % (48, 20))), 96)
