"""GPU: whole-model parity of the H100 engine (through models.Darknet / utils.utils.compute_loss, i.e. the
reference-facing API on top of the C ABI) against the oracle and the committed reference fixtures."""
import numpy as np
import pytest
import torch

from helpers import anchor_vecs, attach_hyp, build_model, golden, module_defs, orc

pytestmark = pytest.mark.gpu

# fp16 activation policy of config C1: documented tolerances vs the fp32 reference (SURVEY.md section 7 / A.9)
BOX_REL_TOL_FP32REF = 3e-2      # xywh, relative to max(|ref|, 1 px)
PROB_ABS_TOL_FP32REF = 1.5e-2   # obj / cls probabilities
# against the oracle that follows the same precision policy (fp16 weights/activations, fp32 accumulate)
BOX_REL_TOL_EMU = 1e-2
PROB_ABS_TOL_EMU = 5e-3


def _errs(got, ref):
    box_rel = ((got[..., :4] - ref[..., :4]).abs() / ref[..., :4].abs().clamp(min=1.0)).max().item()
    prob = (got[..., 4:] - ref[..., 4:]).abs().max().item()
    return box_rel, prob


@pytest.mark.parametrize("name,B,S,seed", [("yolov3-tiny", 2, 96, 3), ("yolov3", 2, 64, 0), ("yolov4", 2, 64, 0),
                                           ("yolov3-tiny", 1, 416, 0)])
def test_eval_forward_parity(name, B, S, seed):
    g = golden("%s_%d_eval" % (name, S))
    model = build_model(name, device="cuda").eval()
    x = orc.synth_images(B, S, S, seed=seed)
    with torch.no_grad():
        io, p, feats = model(x.cuda())
        io2, p2, _ = model(x.cuda())          # second call replays the captured CUDA graph
    torch.cuda.synchronize()
    assert io.shape == g["io"].shape and len(p) == len([k for k in g.files if k.startswith("p")])
    assert torch.equal(io, io2), "CUDA-graph replay differs from the eager launch sequence"
    io = io.cpu()
    # (1) decode is exact given our own raw head outputs: grid/anchor indexing + fp32 math
    ys = [d for d in module_defs(name) if d['type'] == 'yolo']
    strides = orc.yolo_strides(name, len(ys))
    rows = 0
    for d, s, pi in zip(ys, strides, p):
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
        assert torch.equal(cell[..., 0], gx) and torch.equal(cell[..., 1], gy), "grid indices must be bit exact"
    # (2) vs the oracle under the same precision policy
    import models
    from helpers import cfg_path
    sd = orc.synth_state_dict(models.Darknet(cfg_path(name)).state_dict(), 0)
    with torch.no_grad():
        io_emu, _ = orc.darknet_forward(module_defs(name), sd, x, name, emulate_fp16=True)
    be, pe = _errs(io, io_emu)
    # (3) vs the reference's own fp32 output
    bf, pf = _errs(io, torch.from_numpy(g["io"]))
    print("\n[%s %dx%d] vs fp16-policy oracle: box_rel=%.3g prob_abs=%.3g | vs fp32 reference: box_rel=%.3g prob_abs=%.3g"
          % (name, S, S, be, pe, bf, pf))
    assert be <= BOX_REL_TOL_EMU and pe <= PROB_ABS_TOL_EMU
    assert bf <= BOX_REL_TOL_FP32REF and pf <= PROB_ABS_TOL_FP32REF


def test_feature_out_lazy_and_graph_toggle():
    model = build_model("yolov3-tiny", device="cuda").eval()
    x = orc.synth_images(2, 96, 96, seed=3).cuda()
    model.keep_features = True
    with torch.no_grad():
        io, p, feats = model(x)
        f0 = feats[0]
    assert len(feats) == 12 and f0.shape == (2, 16, 96, 96) and f0.dtype == torch.float32
    model.keep_features = None
    model.use_cuda_graph = False
    with torch.no_grad():
        io_b, _, feats_b = model(x)
    torch.testing.assert_close(io, io_b, rtol=2e-3, atol=2e-3)   # shortcut fusion on/off: <= fp16 rounding
    with pytest.raises(RuntimeError):
        feats_b[0]


def test_cpu_input_fails_loudly():
    model = build_model("yolov3-tiny").eval()
    with pytest.raises(RuntimeError):
        model(orc.synth_images(1, 64, 64))


def test_loss_parity_fp32():
    """compute_loss / build_targets through utils.utils on the golden random predictions: fp32, rel 1e-4."""
    from utils import utils as my_utils
    g = golden("loss_case")
    model = attach_hyp(build_model("yolov3", device="cuda"))
    p = [torch.from_numpy(g["p%d" % i]).cuda().requires_grad_(True) for i in range(3)]
    t = torch.from_numpy(g["targets"]).cuda()
    loss, items = my_utils.compute_loss(p, t, model)
    loss.backward()
    np.testing.assert_allclose(items.cpu().numpy(), g["items"], rtol=1e-4)
    for i in range(3):
        np.testing.assert_allclose(p[i].grad.cpu().numpy(), g["dp%d" % i], rtol=1e-4, atol=1e-6)
    tcls, tbox, idx, av = my_utils.build_targets([x.detach() for x in p], t, model)
    for i in range(3):
        assert np.array_equal(torch.stack(idx[i]).cpu().numpy(), g["idx%d" % i]), "indices must be bit exact"
        assert np.array_equal(tcls[i].cpu().numpy(), g["tcls%d" % i])
        np.testing.assert_allclose(tbox[i].cpu().numpy(), g["tbox%d" % i], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(av[i].cpu().numpy(), g["av%d" % i], rtol=1e-6)


def test_loss_edge_cases():
    from utils import utils as my_utils
    model = attach_hyp(build_model("yolov3-tiny", device="cuda"))
    g = torch.Generator().manual_seed(9)
    p = [torch.randn(2, 3, s, s, 85, generator=g).cuda().requires_grad_(True) for s in (2, 4)]
    av = anchor_vecs("yolov3-tiny")
    # no targets at all
    loss, items = my_utils.compute_loss(p, torch.zeros(0, 6).cuda(), model)
    ref, ritems = orc.compute_loss([x.detach().cpu() for x in p], torch.zeros(0, 6), av, model.hyp, 80, 1.0)
    np.testing.assert_allclose(items.cpu().numpy(), ritems.numpy(), rtol=1e-4)
    # duplicates: many targets in the same cell -> last match (anchor-major, target-minor) owns tobj
    t = torch.tensor([[0, 3, 0.26, 0.26, 0.3, 0.4], [0, 5, 0.27, 0.27, 0.3, 0.4], [0, 7, 0.27, 0.26, 0.31, 0.41],
                      [1, 1, 0.8, 0.8, 0.2, 0.1]], dtype=torch.float32)
    pr = [x.detach().cpu().requires_grad_(True) for x in p]
    ref, ritems = orc.compute_loss(pr, t, av, model.hyp, 80, 1.0)
    ref.backward()
    loss, items = my_utils.compute_loss(p, t.cuda(), model)
    loss.backward()
    np.testing.assert_allclose(items.cpu().numpy(), ritems.numpy(), rtol=1e-4)
    for a, b in zip(p, pr):
        np.testing.assert_allclose(a.grad.cpu().numpy(), b.grad.numpy(), rtol=1e-4, atol=1e-6)


def test_uint8_and_fp16_images_match_the_reference_normalisation():
    """uint8 batches are normalised inside the stem kernel with the reference's "/ 256.0" (test.py:95, train.py:348);
    fp16 batches are consumed as they are.  Both must equal the explicit host-side conversion bit for bit."""
    model = build_model("yolov3-tiny", device="cuda").eval()
    g = torch.Generator().manual_seed(5)
    u8 = torch.randint(0, 256, (2, 3, 96, 96), dtype=torch.uint8, generator=g).cuda()
    with torch.no_grad():
        ref_io, ref_p, _ = model(u8.float() / 256.0)
        io, p, _ = model(u8)
        io16, _, _ = model((u8.float() / 256.0).half())
    torch.cuda.synchronize()
    assert torch.equal(io, ref_io)
    assert all(torch.equal(a, b) for a, b in zip(p, ref_p))
    assert torch.equal(io16, ref_io)          # k/256 is exact in fp16


def test_map_on_held_batch_matches_reference():
    """BASELINE north_star: mAP on a held synthetic batch vs the reference.  The held labels are the reference's own
    detections on the batch (map_case.npz, produced by running the reference); the engine's predictions go through the
    same NMS / matching / AP pipeline (oracle/metrics_oracle.py, pinned to the reference's).  With random weights the
    ~2800 candidates sit densely around the confidence threshold, so ONE detection flipping in or out moves the mean AP
    by ~1.5e-4: the fp32-vs-fp16-policy oracle pair shows exactly that.  Gate: 5e-3 (measured 2.6e-3), or 3x the deviation
    the precision policy itself causes (measured with the oracle in this test) if that is larger; the 1e-4 of the
    north star is reached only when no candidate straddles a threshold, which fp16 activations cannot guarantee."""
    from oracle import metrics_oracle as mo
    import models as _models
    from helpers import cfg_path
    g = golden("map_case")
    S, B = int(g["size"]), g["inf_out"].shape[0]
    conf, iou = float(g["conf_thres"]), float(g["iou_thres"])
    model = build_model("yolov3-tiny", device="cuda").eval()
    x = orc.synth_images(B, S, S, seed=int(g["seed"]))
    with torch.no_grad():
        io, _, _ = model(x.cuda())
    torch.cuda.synchronize()
    labels = [torch.from_numpy(g["labels%d" % i]) for i in range(B)]
    m50, m, n = mo.mean_ap(io, labels, conf, iou, S, S)
    sd = orc.synth_state_dict(_models.Darknet(cfg_path("yolov3-tiny")).state_dict(), 0)
    with torch.no_grad():
        io_pol, _ = orc.darknet_forward(module_defs("yolov3-tiny"), sd, x, "yolov3-tiny", emulate_fp16=True)
    y50, y, yn = mo.mean_ap(io_pol, labels, conf, iou, S, S)
    r50, r = float(g["map50"]), float(g["map"])
    print("\n[mAP held batch] reference %.6f / %.6f (%d labels) | engine %.6f / %.6f (%d det) | fp16-policy oracle "
          "%.6f / %.6f (%d det)" % (r50, r, sum(l.shape[0] for l in labels), m50, m, n, y50, y, yn))
    # one flipped detection out of ~2800 moves the mean AP by ~1.5e-4 (the oracle pair above differs by exactly one);
    # the engine's probabilities are within 1e-3 of the reference's, i.e. a handful of threshold flips are expected
    tol50 = max(1e-4, 3 * abs(y50 - r50), 5e-3)
    tol = max(1e-4, 3 * abs(y - r), 5e-3)
    assert abs(m50 - r50) <= tol50, (m50, r50, y50)
    assert abs(m - r) <= tol, (m, r, y)
    assert abs(n - sum(l.shape[0] for l in labels)) <= 0.01 * n


SLICED_CFG = """
[net]
width=64
height=64
channels=3

[convolutional]
batch_normalize=1
filters=32
size=3
stride=1
pad=1
activation=leaky

[convolutional]
batch_normalize=1
filters=64
size=3
stride=1
pad=1
activation=leaky

[convolutional]
batch_normalize=1
filters=64
size=1
stride=1
pad=1
activation=leaky

[shortcut]
from=-3
activation=linear

[convolutional]
batch_normalize=1
filters=32
size=1
stride=1
pad=1
activation=leaky

[shortcut]
from=-3
activation=linear

[convolutional]
batch_normalize=1
filters=64
size=3
stride=2
pad=1
activation=leaky

[convolutional]
filters=255
size=1
stride=1
pad=1
activation=linear

[yolo]
mask = 0,1,2
anchors = 10,13, 16,30, 33,23, 30,61, 62,45, 59,119, 116,90, 156,198, 373,326
classes=80
num=9
"""


def test_channel_sliced_shortcuts():
    """utils/layers.py:57-72: a shortcut whose addend is narrower (the sum covers its channels, the rest of x passes
    through) or wider (only its first channels are added) than x -- inference and training plans against the oracle."""
    import os
    import tempfile
    import models
    from utils.parse_config import parse_model_cfg
    from utils import utils as my_utils
    d = tempfile.mkdtemp(prefix="b2y_sliced_")
    path = os.path.join(d, "sliced-yolov3.cfg")
    with open(path, "w") as f:
        f.write(SLICED_CFG)
    defs = parse_model_cfg(path)[1:]
    m = models.Darknet(path)
    sd = orc.synth_state_dict(m.state_dict(), 0)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    x = orc.synth_images(2, 64, 64, seed=4)
    with torch.no_grad():
        io, p, _ = m(x.cuda())
        ref, _ = orc.darknet_forward(defs, sd, x, "yolov3", emulate_fp16=True)
    b, pr = _errs(io.cpu(), ref)
    print("\n[sliced shortcuts eval] box_rel=%.3g prob_abs=%.3g" % (b, pr))
    assert b < 5e-3 and pr < 2e-3
    # training step: loss and gradient norms against the fp32 oracle
    m = attach_hyp(m).train()
    t = orc.synth_targets(2, 6, 80, seed=1)
    pred, _ = m(x.cuda())
    loss, items = my_utils.compute_loss(pred, t.cuda(), m)
    loss.backward()
    sdr = {k: (v.clone().requires_grad_(True) if v.dtype.is_floating_point and not k.endswith(("running_mean", "running_var")) else v.clone())
           for k, v in orc.synth_state_dict(models.Darknet(path).state_dict(), 0).items()}
    pe, _ = orc.darknet_forward(defs, sdr, x, "yolov3", training=True)
    ys = [dd for dd in defs if dd['type'] == 'yolo']
    av = [m.module_list[j].anchor_vec.detach().float().cpu() for j in m.yolo_layers]   # the model's own anchors / stride
    le, ie = orc.compute_loss(pe, t, av, dict(m.hyp), 80, 1.0)
    le.backward()
    rel = [abs(float(pp.grad.norm()) - float(sdr[k].grad.norm())) / (float(sdr[k].grad.norm()) + 1e-6)
           for k, pp in m.named_parameters()]
    print("[sliced shortcuts train] loss %.5f vs %.5f, grad-norm rel median %.3g worst %.3g"
          % (float(loss), float(le), float(np.median(rel)), max(rel)))
    assert abs(float(loss) - float(le)) / abs(float(le)) < 1e-2
    assert float(np.median(rel)) < 2e-2


@pytest.mark.parametrize("name,B,S,seed", [("yolov3-tiny", 1, 416, 0), ("yolov3", 2, 64, 0), ("yolov4", 2, 64, 0)])
def test_accurate_mode_matches_fp32_reference(name, B, S, seed):
    """model.accurate = True: split-fp16 tensor-core convolutions with fp32 activations (b200yolo/accurate.py).
    north_star: "fp32 loss and box coords within 1e-4 rel" against the reference's own fp32 output."""
    g = golden("%s_%d_eval" % (name, S))
    model = build_model(name, device="cuda").eval()
    model.accurate = True
    x = orc.synth_images(B, S, S, seed=seed)
    with torch.no_grad():
        io, p, _ = model(x.cuda())
    torch.cuda.synchronize()
    b, pr = _errs(io.cpu(), torch.from_numpy(g["io"]))
    print("\n[%s %dx%d accurate mode] vs fp32 reference: box_rel=%.3g prob_abs=%.3g" % (name, S, S, b, pr))
    assert b <= 1e-4 and pr <= 1e-4


def test_map_on_held_batch_accurate_mode():
    """BASELINE north_star: mAP on a held synthetic batch within 1e-4 of the reference -- in the fp32-accurate mode."""
    from oracle import metrics_oracle as mo
    g = golden("map_case")
    S, B = int(g["size"]), g["inf_out"].shape[0]
    conf, iou = float(g["conf_thres"]), float(g["iou_thres"])
    model = build_model("yolov3-tiny", device="cuda").eval()
    model.accurate = True
    x = orc.synth_images(B, S, S, seed=int(g["seed"]))
    with torch.no_grad():
        io, _, _ = model(x.cuda())
    torch.cuda.synchronize()
    labels = [torch.from_numpy(g["labels%d" % i]) for i in range(B)]
    m50, m, n = mo.mean_ap(io, labels, conf, iou, S, S)
    r50, r = float(g["map50"]), float(g["map"])
    dmax = float((io.cpu() - torch.from_numpy(g["inf_out"])).abs().max())
    print("\n[mAP held batch, accurate mode] reference %.6f / %.6f | engine %.6f / %.6f (%d det) | max |io - ref| %.3g"
          % (r50, r, m50, m, n, dmax))
    assert abs(m50 - r50) <= 1e-4 and abs(m - r) <= 1e-4
