"""GPU: channel-pruned models (widths such as 1, 3, 37, 100) on the fp16 eval plan, against the reference's fp32 outputs
in tests/golden/pruned_case.npz (oracle/gen_golden_pruned.py) and the fp16-policy oracle, with the same gate as the
stock eval fixtures in test_gpu_model.py; and the graphs that do not run pruned widths refuse them by name."""
import numpy as np
import pytest
import torch

from helpers import orc
from pruned_models import build_pruned, cases, compact_defs, fixture, images

pytestmark = pytest.mark.gpu

CASES = [n for n, _ in cases()]
BOX_REL_TOL_FP32REF = 3e-2
PROB_ABS_TOL_FP32REF = 1.5e-2
BOX_REL_TOL_EMU = 1e-2
PROB_ABS_TOL_EMU = 5e-3


def _errs(got, ref):
    box_rel = ((got[..., :4] - ref[..., :4]).abs() / ref[..., :4].abs().clamp(min=1.0)).max().item()
    prob = (got[..., 4:] - ref[..., 4:]).abs().max().item()
    return box_rel, prob


@pytest.mark.parametrize("name", CASES)
def test_pruned_eval_matches_reference(name):
    model = build_pruned(name, device="cuda").eval()
    x = images(name)
    ref = torch.from_numpy(fixture()[name + ":io"])
    sd = {k: v.cpu() for k, v in model.state_dict().items()}
    with torch.no_grad():
        io_emu, _ = orc.darknet_forward(compact_defs(name)[1:], sd, x, name, emulate_fp16=True)
    for graph in (True, False):
        model.use_cuda_graph = graph
        for xin in (x.cuda(), (x * 256).round().to(torch.uint8).cuda()):
            with torch.no_grad():
                io, p, _ = model(xin)
                io2, _, _ = model(xin)           # with graphs on: the replay of the captured graph
            torch.cuda.synchronize()
            assert torch.equal(io, io2)
            io = io.cpu()
            assert io.shape == ref.shape
            # grid / anchor decode is exact given our own raw head outputs
            rows = 0
            ys = [d for d in model.module_defs if d['type'] == 'yolo']
            for d, s, pi in zip(ys, orc.yolo_strides(name, len(ys)), p):
                pi = pi.cpu()
                Bq, na, ny, nx, no = pi.shape
                raw = pi.permute(0, 1, 4, 2, 3).reshape(Bq, na * no, ny, nx)
                io_ref, _ = orc.yolo_layer(raw, np.asarray(d['anchors'])[d['mask']], s, int(d['classes']), False)
                mine = io[:, rows:rows + na * ny * nx]
                rows += na * ny * nx
                torch.testing.assert_close(mine, io_ref, rtol=1e-5, atol=1e-5)
                cell = torch.round(mine.view(Bq, na, ny, nx, no)[..., :2] / s - torch.sigmoid(pi[..., :2]))
                gx = torch.arange(nx).view(1, 1, 1, nx).expand(Bq, na, ny, nx).float()
                gy = torch.arange(ny).view(1, 1, ny, 1).expand(Bq, na, ny, nx).float()
                assert torch.equal(cell[..., 0], gx) and torch.equal(cell[..., 1], gy)
            be, pe = _errs(io, io_emu)
            bf, pf = _errs(io, ref)
            print("\n[pruned %s graph=%s %s] vs fp16-policy oracle: box_rel=%.3g prob_abs=%.3g | vs fp32 reference: "
                  "box_rel=%.3g prob_abs=%.3g" % (name, graph, xin.dtype, be, pe, bf, pf))
            assert be <= BOX_REL_TOL_EMU and pe <= PROB_ABS_TOL_EMU
            assert bf <= BOX_REL_TOL_FP32REF and pf <= PROB_ABS_TOL_FP32REF


@pytest.mark.parametrize("name", CASES)
def test_pruned_feature_out_has_logical_widths(name):
    from b200yolo.layout import feature_slots
    model = build_pruned(name, device="cuda").eval()
    model.keep_features = True
    x = images(name)
    with torch.no_grad():
        _, _, feats = model(x.cuda())
        got = [feats[j].cpu() for j in range(len(feats))]
    sd = {k: v.cpu() for k, v in model.state_dict().items()}
    with torch.no_grad():
        outs = orc.darknet_forward(compact_defs(name)[1:], sd, x, name, emulate_fp16=True, return_layers=True)
    slots = feature_slots(model)
    assert len(got) == len(slots)
    worst = 0.0
    for f, i in zip(got, slots):
        assert f.shape == outs[i].shape, (i, f.shape, outs[i].shape)
        worst = max(worst, ((f - outs[i]).abs().max() / outs[i].abs().max().clamp(min=1.0)).item())
    print("\n[pruned %s feature_out] worst relative error %.3g" % (name, worst))
    assert worst < 2e-2


def test_graphs_without_pruned_widths_refuse_them_by_layer():
    import models
    x = images("yolov3").cuda()
    # training plan
    model = build_pruned("yolov3", device="cuda").train()
    with pytest.raises(NotImplementedError, match=r"layer \d+: BatchNorm training needs a multiple of 8"):
        model(x)
    # fp32-accurate mode
    model = build_pruned("yolov3-tiny", device="cuda").eval()
    model.accurate = True
    with pytest.raises(NotImplementedError, match=r"layer \d+: \d+ channels; the accurate mode"):
        with torch.no_grad():
            model(images("yolov3-tiny").cuda())
    # INT8 graph
    qm = models.Darknet(compact_defs("yolov3"), quantized=3, shortcut_way=1).cuda().eval()
    with pytest.raises(NotImplementedError, match=r"layer \d+: int8 graph needs"):
        with torch.no_grad():
            qm(x)
