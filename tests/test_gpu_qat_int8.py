"""GPU: the eval forward of google-QAT (quantized=1) models as the captured INT8 graph (b200yolo/qengine.py QPlan), which
must equal the QAT module forwards (b200yolo/qat.py QatRunner) bit for bit, re-pack itself after training, and be taken
only by the models qengine.int8_graph_refusal accepts; plus the int8 max-pool kernel it needs (b2y_maxpool_i8)."""
import os
import tempfile

import pytest
import torch
import torch.nn.functional as F

from helpers import attach_hyp, cfg_path, orc

pytestmark = pytest.mark.gpu

STEPS = 100

# ---------------------------------------------------------------------------------------------------------------------
# b2y_maxpool_i8


def _maxpool_i8(x, x_pitch, y, y_pitch, B, H, W, C, k, s, pad_mode):
    from b200yolo.lib import call, ptr, stream_ptr
    call("b2y_maxpool_i8", ptr(x), x_pitch, ptr(y), y_pitch, B, H, W, C, k, s, pad_mode, stream_ptr())


def _pool_case(B, H, W, C, k, s, tiny, gen):
    """codes in a buffer wider than C (x_pitch = C + 16), the result written into a channel slot at offset 16 of a
    buffer of pitch C + 32; the channels around the slot must keep their sentinel"""
    xb = torch.randint(-128, 128, (B, H, W, C + 16), generator=gen, dtype=torch.int8).cuda()
    x = xb[..., :C]
    xf = x.permute(0, 3, 1, 2).float()
    ref = F.max_pool2d(F.pad(xf, (0, 1, 0, 1)), 2, 1) if tiny else F.max_pool2d(xf, k, s, (k - 1) // 2)
    ref = ref.permute(0, 2, 3, 1).to(torch.int8)
    Ho, Wo = ref.shape[1], ref.shape[2]
    yb = torch.full((B, Ho, Wo, C + 32), 77, dtype=torch.int8, device="cuda")
    _maxpool_i8(x, C + 16, yb[..., 16:], C + 32, B, H, W, C, k, s, 1 if tiny else 0)
    torch.cuda.synchronize()
    assert torch.equal(yb[..., 16:16 + C], ref), (B, H, W, C, k, s, tiny)
    assert bool((yb[..., :16] == 77).all()) and bool((yb[..., 16 + C:] == 77).all())


@pytest.mark.parametrize("k,s,tiny", [(2, 2, False), (2, 1, True), (5, 1, False), (9, 1, False), (13, 1, False)])
def test_maxpool_i8_matches_torch(k, s, tiny):
    """yolov3-tiny's 2x2 stride-2 pool, its zero-padded 2x2 stride-1 pool and the SPP pools, on odd and even maps (the
    SPP shapes on both the shared-memory plane kernel and, above 32 x 32 pixels, the direct-window one)"""
    gen = torch.Generator().manual_seed(k * 10 + s)
    cases = [(1, 13, 13, 16), (32, 13, 13, 64), (1, 7, 5, 1024), (32, 7, 5, 32), (2, 26, 26, 256), (1, 1, 1, 16),
             (2, 40, 33, 48)]
    for B, H, W, C in cases:
        if H < k and s > 1:
            continue                # no output pixel: torch refuses the shape, b2y_maxpool_i8 returns B2Y_ERR_INVALID
        _pool_case(B, H, W, C, k, s, tiny, gen)


def test_maxpool_i8_rejects_bad_arguments():
    """bad shapes, pitches, alignment or modes return B2Y_ERR_INVALID and launch nothing (the output keeps its bytes)"""
    from b200yolo.lib import B2YError
    x = torch.zeros((1, 8, 8, 64), dtype=torch.int8, device="cuda")
    y = torch.full((1, 8, 8, 64), 5, dtype=torch.int8, device="cuda")
    bad = [
        dict(C=8, xp=64, yp=64),                    # channels not a multiple of 16
        dict(C=64, xp=48, yp=64),                   # x pitch narrower than C
        dict(C=32, xp=64, yp=40),                   # y pitch not a multiple of 16
        dict(C=32, xp=64, yp=64, pad_mode=2),       # unknown pad mode
        dict(C=32, xp=64, yp=64, k=0),
        dict(C=32, xp=64, yp=64, s=0),
        dict(C=32, xp=64, yp=64, k=20, pad_mode=1),  # window larger than the padded map
        dict(C=32, xp=64, yp=64, H=0),
        dict(C=32, xp=64, yp=64, misalign=True),    # 16-byte vectors need 16-byte aligned tensors
    ]
    for b in bad:
        xx = x.view(-1)[1:].as_strided((1, 8, 8, 32), (4096, 512, 64, 1)) if b.get('misalign') else x
        with pytest.raises(B2YError):
            _maxpool_i8(xx, b['xp'], y, b['yp'], 1, b.get('H', 8), 8, b['C'], b.get('k', 2), b.get('s', 2),
                        b.get('pad_mode', 0))
    with pytest.raises(B2YError):
        from b200yolo.lib import call, stream_ptr
        call("b2y_maxpool_i8", None, 64, None, 64, 1, 8, 8, 64, 2, 2, 0, stream_ptr())
    torch.cuda.synchronize()
    assert bool((y == 5).all())


# ---------------------------------------------------------------------------------------------------------------------
# models


def _spp_cfg():
    """yolov3-spp: yolov3 with the SPP block (max-pools 5 / 9 / 13 and their concat) in the first head"""
    from b200yolo import cfggen as g
    c = g._Cfg(g._net())
    c.conv(32, 3)
    for filters, blocks in ((64, 1), (128, 2), (256, 8), (512, 8), (1024, 4)):
        c.conv(filters, 3, 2)
        for _ in range(blocks):
            c.conv(filters // 2, 1)
            c.conv(filters, 3)
            c.shortcut(-3)
    for scale, (mid, mask, skip) in enumerate(((512, (6, 7, 8), None), (256, (3, 4, 5), 61), (128, (0, 1, 2), 36))):
        if skip is not None:
            c.route(-4)
            c.conv(mid, 1)
            c.upsample(2)
            c.route(-1, skip)
        for j in range(3):
            c.conv(mid, 1)
            if scale == 0 and j == 1:
                c.maxpool(5, 1)
                c.route(-2)
                c.maxpool(9, 1)
                c.route(-4)
                c.maxpool(13, 1)
                c.route(-1, -3, -5, -6)
                c.conv(mid, 1)
            c.conv(mid * 2, 3)
        c.conv(255, 1, act="linear", bn=0)
        c.yolo(mask, g.COCO_ANCHORS_V3, 80, 9, (("random", 1),))
    return c.text()


def _grouped_route_cfg():
    """a small detector with a yolov4-tiny style grouped route (the upper channel half of the layer before it)"""
    from b200yolo import cfggen as g
    c = g._Cfg(g._net())
    c.conv(32, 3, 2)
    c.conv(64, 3, 2)
    c.block("route", ("layers", -1), ("groups", 2), ("group_id", 1))
    c.conv(32, 3)
    c.route(-1, -2)
    c.maxpool(2, 2)
    c.conv(128, 3)
    c.conv(255, 1, act="linear", bn=0)
    c.yolo((3, 4, 5), g.TINY_ANCHORS, 80, 6)
    return c.text()


_EXTRA_CFGS = {"yolov3-spp": _spp_cfg, "grouped-route": _grouped_route_cfg}
_CFG_DIR = tempfile.mkdtemp(prefix="b2y_q1_cfg_")


def _cfg(name):
    if name not in _EXTRA_CFGS:
        return cfg_path(name)
    path = os.path.join(_CFG_DIR, name + ".cfg")
    if not os.path.exists(path):
        with open(path, "w") as f:
            f.write(_EXTRA_CFGS[name]())
    return path


def _qat_model(name, way=1, a_bit=8):
    """quantized=1 Darknet with the synthetic float parameters of oracle.synth_state_dict (as tests/test_gpu_qat.py)"""
    import models
    fm = models.Darknet(_cfg(name))
    sd = orc.synth_state_dict(fm.state_dict(), 0)
    qm = models.Darknet(_cfg(name), quantized=1, a_bit=a_bit, w_bit=8, shortcut_way=way, steps=STEPS)
    with torch.no_grad():
        for i, m in enumerate(qm.module_list):
            pre = 'module_list.%d.' % i
            if m.__class__.__name__ != 'Sequential' or not len(m):
                continue
            if hasattr(m[0], 'activation_quantizer'):
                c = m[0]
                c.weight.copy_(sd[pre + 'Conv2d.weight'])
                if (pre + 'BatchNorm2d.weight') in sd:
                    c.gamma.copy_(sd[pre + 'BatchNorm2d.weight'])
                    c.beta.copy_(sd[pre + 'BatchNorm2d.bias'])
                else:
                    c.bias.copy_(sd[pre + 'Conv2d.bias'])
            else:       # the float [depthwise] / [se] blocks of a google-QAT MobileNet
                for n, t in m.state_dict().items():
                    if (pre + n) in sd:
                        t.copy_(sd[pre + n])
    return attach_hyp(qm.cuda())


def _train(qm, steps, seed=0):
    """QAT training steps on the engine at 64 x 64, batch 2: they set the quantiser scales and running statistics"""
    from utils import utils as my_utils
    qm.train()
    opt = torch.optim.SGD(qm.parameters(), lr=1e-3, momentum=0.9)
    for k in range(steps):
        x = orc.synth_images(2, 64, 64, seed=seed + k).cuda()
        t = orc.synth_targets(2, 6, 80, seed=seed + k + 1).cuda()
        pred, _ = qm(x)
        loss, _ = my_utils.compute_loss(pred, t, qm)
        opt.zero_grad()
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    qm.eval()


def _runner_eval(qm, x):
    from b200yolo.qat import QatRunner
    with torch.no_grad():
        io, p, _ = QatRunner(qm).forward(x)
    return io.clone(), [t.clone() for t in p]


def _q1_plans(qm):
    return [k for k in qm.engine().plans if len(k) == 3 and k[1] == 'q1']


def _assert_same(got, ref, what):
    io, p = got[0], got[1]
    assert torch.equal(io, ref[0]), "%s: io differs in %d of %d values" % (what, int((io != ref[0]).sum()), io.numel())
    assert len(p) == len(ref[1])
    for j, (a, b) in enumerate(zip(p, ref[1])):
        assert torch.equal(a, b), "%s: p%d differs in %d of %d values" % (what, j, int((a != b).sum()), a.numel())


def _check_sizes(qm, name, sizes):
    from b200yolo.qengine import int8_graph_refusal
    assert int8_graph_refusal(qm) is None
    for (h, w) in sizes:
        x = orc.synth_images(2, h, w, seed=h + w).cuda()
        ref = _runner_eval(qm, x)
        for graph in (True, False):
            qm.use_cuda_graph = graph
            with torch.no_grad():
                for call in range(2):          # graph: the eager first call, then the capture and its replay
                    io, p, _ = qm(x)
                    _assert_same((io, p), ref, "%s %dx%d graph=%s call %d" % (name, h, w, graph, call))
        qm.use_cuda_graph = True
    assert len(_q1_plans(qm)) == len(sizes)


@pytest.mark.parametrize("way", [1, 2])
@pytest.mark.parametrize("name", ["yolov3", "yolov3-tiny", "yolov3-spp"])
def test_qat_int8_graph_equals_module_forwards(name, way):
    """io and every p of the INT8 graph == QatRunner's eval outputs, captured and eager, square and rectangular"""
    qm = _qat_model(name, way)
    _train(qm, 2)
    _check_sizes(qm, name, [(64, 64), (416, 416), (256, 416)])


@pytest.mark.parametrize("way", [1, 2])
def test_qat_int8_graph_unfused_shortcuts(way):
    """the stand-alone shortcut launches (b2y_qshortcut_i8, and the clamped addends of QuantizedShortcut_max through
    b2y_requant_i8) instead of the shortcut folded into the conv epilogue, captured and eager"""
    from b200yolo.qengine import QPlan, int8_graph_refusal
    qm = _qat_model("yolov3", way)
    _train(qm, 2)
    assert int8_graph_refusal(qm) is None
    x = orc.synth_images(2, 64, 64, seed=128).cuda()
    ref = _runner_eval(qm, x)
    plan = QPlan(qm, tuple(x.shape), x.device, fuse_shortcuts=False)
    assert not any(st.kind == 'conv' and st.shortcut for st in plan.steps)
    for graph in (True, False):
        qm.use_cuda_graph = graph
        with torch.no_grad():
            for call in range(2):          # graph: the eager first call, then the capture and its replay
                io, p, _ = plan.forward(x)
                _assert_same((io, p), ref, "yolov3 unfused graph=%s call %d" % (graph, call))
    qm.use_cuda_graph = True


def test_qat_int8_plan_follows_training():
    """three training steps, eval, three more, eval: each eval equals a fresh QatRunner eval, so the weight, running
    statistics and (re-assigned) scale changes re-pack the cached plan and re-capture its graph"""
    qm = _qat_model("yolov3-tiny", 1)
    x = orc.synth_images(4, 96, 96, seed=11).cuda()
    outs = []
    for round_ in range(2):
        _train(qm, 3, seed=100 * round_)
        ref = _runner_eval(qm, x)
        with torch.no_grad():
            for call in range(3):
                io, p, _ = qm(x)
                _assert_same((io, p), ref, "round %d call %d" % (round_, call))
        outs.append(io.clone())
        assert len(_q1_plans(qm)) == 1
    assert not torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("name,a_bit,why", [("yolov3-mobilenet", 8, "'depthwise'"), ("yolov3-tiny", 16, "a_bit 16"),
                                            ("grouped-route", 8, "grouped route")])
def test_qat_models_outside_the_rule_keep_the_module_forwards(name, a_bit, why):
    from b200yolo.qengine import int8_graph_refusal
    qm = _qat_model(name, 1, a_bit=a_bit)
    reason = int8_graph_refusal(qm)
    assert reason is not None and why in reason, reason
    qm.train()
    with torch.no_grad():                       # a training-mode forward sets the quantiser scales
        qm(orc.synth_images(2, 64, 64, seed=1).cuda())
    qm.eval()
    x = orc.synth_images(2, 64, 64, seed=2).cuda()
    ref = _runner_eval(qm, x)
    with torch.no_grad():
        io, p, _ = qm(x)
    _assert_same((io, p), ref, name)
    assert not _q1_plans(qm)
