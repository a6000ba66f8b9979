"""GPU: parity at the BASELINE sizes (640x640) -- the plans, tile schedules and CTA-pair / weight-stationary kernel
variants the benchmark actually runs -- against fixtures produced by the reference itself on CPU fp32
(oracle/gen_golden_640.py) and against the oracle run live under the engine's precision policy.

  * yolov3 / yolov4 inference: the engine runs the BASELINE batch (32 images); its first two images are the fixture's.
  * yolov4 training step, 8 images = the per-GPU slice of BASELINE configs[2]: loss items, sampled predictions, the
    gradient of EVERY parameter (element-wise against the fp16-policy oracle, norms against the fp32 reference),
    BatchNorm running statistics.

Every gate below is a constant; the test prints the measured errors.
"""
import numpy as np
import pytest
import torch

from helpers import anchor_vecs, attach_hyp, build_model, cfg_path, golden, module_defs, orc

pytestmark = pytest.mark.gpu

SIZE = 640
# ---- inference, fp16 activation policy (config C1).  Gates against the fp32 reference and the fp16-policy oracle:
# (yolov3's leaky network with the synthetic weights is the less well conditioned of the two: two different roundings of
#  the same fp16 policy (mkldnn's fp32 accumulation order vs the tensor core's) end up far apart.)
TOL = {"yolov3": {"box_ref": 1.8e-2, "prob_ref": 5.6e-3, "box_emu": 3.0e-2, "prob_emu": 8.8e-3},
       "yolov4": {"box_ref": 4.4e-4, "prob_ref": 1.8e-4, "box_emu": 8.0e-4, "prob_emu": 1.7e-4}}


def _errs(got, ref):
    box_rel = ((got[..., :4] - ref[..., :4]).abs() / ref[..., :4].abs().clamp(min=1.0)).max().item()
    prob = (got[..., 4:] - ref[..., 4:]).abs().max().item()
    return box_rel, prob


def _state(name):
    import models
    return orc.synth_state_dict(models.Darknet(cfg_path(name)).state_dict(), 0)


@pytest.mark.parametrize("name", ["yolov3", "yolov4"])
def test_eval_forward_640_bs32(name):
    g = golden("%s_640_eval" % name)
    model = build_model(name, device="cuda").eval()
    x2 = orc.synth_images(2, SIZE, SIZE, seed=0)                 # the fixture's two images
    x = torch.cat([x2, orc.synth_images(30, SIZE, SIZE, seed=5)], 0)
    with torch.no_grad():
        io, p, _ = model(x.cuda())
        io_b, _, _ = model(x.cuda())                             # CUDA-graph replay
    torch.cuda.synchronize()
    assert tuple(io.shape) == (32, 25200, 85)
    assert torch.equal(io, io_b)
    io2 = io[:2].cpu()
    rows = g["rows"]
    # grid / anchor indexing: bit exact on every cell of the 32 images (decode recomputed from our raw outputs)
    ys = [d for d in module_defs(name) if d['type'] == 'yolo']
    strides = orc.yolo_strides(name, len(ys))
    off = 0
    for d, s, pi in zip(ys, strides, p):
        Bq, na, ny, nx, no = pi.shape
        mine = io[:, off:off + na * ny * nx].view(Bq, na, ny, nx, no)
        cell = torch.round(mine[..., :2] / s - torch.sigmoid(pi[..., :2]))
        gx = torch.arange(nx, device=io.device).view(1, 1, 1, nx).expand(Bq, na, ny, nx).float()
        gy = torch.arange(ny, device=io.device).view(1, 1, ny, 1).expand(Bq, na, ny, nx).float()
        assert torch.equal(cell[..., 0], gx) and torch.equal(cell[..., 1], gy), "grid indices must be bit exact"
        off += na * ny * nx
    bf, pf = _errs(io2[:, rows], torch.from_numpy(g["io_rows"]))
    with torch.no_grad():
        io_emu, _ = orc.darknet_forward(module_defs(name), _state(name), x2, name, emulate_fp16=True)
    be, pe = _errs(io2, io_emu)
    print("\n[%s 640x640 bs32] vs fp32 reference (sampled rows): box_rel=%.3g prob_abs=%.3g | vs fp16-policy oracle "
          "(all rows): box_rel=%.3g prob_abs=%.3g" % (name, bf, pf, be, pe))
    tol = TOL[name]
    assert bf <= tol["box_ref"] and pf <= tol["prob_ref"]
    assert be <= tol["box_emu"] and pe <= tol["prob_emu"]
    # float64 checksum of the whole output of both images (size-independent property)
    got_sum = io2.double().sum(dim=(1, 2)).numpy()
    np.testing.assert_allclose(got_sum, g["io_sum"], rtol=2e-4)


# ---- training step (config C2 per-GPU slice).  The fp16-activation policy perturbs a randomly initialised 110-layer
# network chaotically less at batch 8 x 640^2 than at the toy sizes (every BatchNorm sees >= 3200 samples), so absolute
# gates are possible:
def test_train_step_640_bs8():
    from utils import utils as my_utils
    name = "yolov4"
    g = golden("yolov4_640_train")
    model = attach_hyp(build_model(name, device="cuda")).train()
    x = orc.synth_images(8, SIZE, SIZE, seed=0)
    t = orc.synth_targets(8, 8, 80, seed=1)
    outs = []
    for it in range(3):                       # eager, graph capture, graph replay: all three must agree
        model.zero_grad(set_to_none=True)
        pred, _ = model(x.cuda())
        loss, items = my_utils.compute_loss(pred, t.cuda(), model)
        loss.backward()
        outs.append((float(loss.detach()), items.detach().cpu().clone()))
        if it == 0:
            params = dict(model.named_parameters())
            grads = {k: p.grad.detach().float().cpu().clone() for k, p in params.items()}
            preds = [pi.detach().cpu().clone() for pi in pred]
            msd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.endswith(("running_mean", "running_var"))}
    torch.cuda.synchronize()
    assert all(np.isfinite(o[0]) for o in outs)
    assert max(abs(o[0] - outs[0][0]) / abs(outs[0][0]) for o in outs) < 2e-3, [o[0] for o in outs]

    # (a) vs the reference's own fp32 step
    items_rel = float((np.abs(outs[0][1].numpy() - g["items"]) / np.abs(g["items"])).max())
    p_abs = max(float((pi.reshape(8, -1, 85)[:, ::29] - torch.from_numpy(g["p%d_rows" % i])).abs().max())
                for i, pi in enumerate(preds))
    names = [str(n) for n in g["grad_names"]]
    ref_norm = dict(zip(names, g["grad_norms"]))
    norm_rel = np.array([abs(float(grads[k].norm()) - ref_norm[k]) / (ref_norm[k] + 1e-8) for k in names])
    elem = []
    for k in names:
        if ("grad::" + k) in g.files:
            ref = torch.from_numpy(g["grad::" + k])
            elem.append(float((grads[k] - ref).abs().max() / ref.abs().max().clamp(min=1e-12)))
    stat_err = max(float((msd[k[6:]] - torch.from_numpy(g[k])).abs().max()) for k in g.files if k.startswith("stat::"))

    # (b) vs the oracle under the engine's forward precision policy, ALL parameters element-wise
    sd = _state(name)
    for k, v in sd.items():
        if v.dtype.is_floating_point and not k.endswith(('running_mean', 'running_var')):
            v.requires_grad_(True)
    pe, _ = orc.darknet_forward(module_defs(name), sd, x, name, training=True, emulate_fp16=True)
    le, ie = orc.compute_loss(pe, t, anchor_vecs(name), dict(orc.DEFAULT_HYP), 80, 1.0)
    le.backward()
    pol = np.array([float((grads[k] - sd[k].grad).norm() / (sd[k].grad.norm() + 1e-12)) for k in names])
    yard = np.array([abs(float(sd[k].grad.norm()) - ref_norm[k]) / (ref_norm[k] + 1e-8) for k in names])
    yard_items = float((np.abs(ie.detach().numpy() - g["items"]) / np.abs(g["items"])).max())
    print("\n[yolov4 train 8x640x640] vs fp32 reference: loss items rel %.3g (policy oracle itself: %.3g) | sampled p abs "
          "%.3g | grad-norm rel median %.3g worst %.3g (policy oracle: %.3g / %.3g) | BN + bias grads element-wise worst "
          "%.3g | running stats abs %.3g || vs fp16-policy oracle, every parameter: rel L2 error median %.3g worst %.3g"
          % (items_rel, yard_items, p_abs, np.median(norm_rel), norm_rel.max(), np.median(yard), yard.max(),
             max(elem), stat_err, np.median(pol), pol.max()))
    # The element-wise figures are printed for
    # the record only: the oracle pair (fp32 vs fp16 policy, CPU) itself is uncorrelated on this batch (relative L2
    # error 1.12 median, oracle/README note in DESIGN.md section 4), so they cannot be gated end to end -- the
    # element-wise gates for every parameter are in test_train_step_layerwise below.
    p_rms = max(float((pi.reshape(8, -1, 85)[:, ::29] - torch.from_numpy(g["p%d_rows" % i])).pow(2).mean().sqrt())
                for i, pi in enumerate(preds))
    print("sampled p rms diff %.3g" % p_rms)
    assert items_rel < 1.8e-2            # measured 8.7e-3 (policy oracle: 1.4e-3)
    assert p_rms < 0.6                   # oracle pair: 0.10 / 0.18 / 0.26 per head on predictions of rms 0.73
    assert np.median(norm_rel) < 4e-2 and norm_rel.max() < 0.6      # measured 1.95e-2 / 0.30 (policy oracle 2.07e-2 / 0.27)
    assert stat_err < 4e-3               # measured 1.8e-3


# ---- layer-wise ("teacher-forced") gates at the BASELINE size ---------------------------------------------------------
# End to end, a randomly initialised 110-layer network with batch-statistics BatchNorm amplifies 16-bit rounding
# chaotically: the ORACLE PAIR (fp32 vs the fp16 activation policy, both on CPU) already disagrees by a relative L2
# error of 1.12 (median over all parameters; 0.10-0.26 rms on predictions of rms 0.73) on this very batch, so no
# element-wise end-to-end gate can be tighter than "uncorrelated".  What CAN be pinned absolutely is every layer of the
# step on the tensors the engine itself produced at 8 x 640 x 640: conv forward, BatchNorm forward, BatchNorm backward,
# weight gradient and (where the input has a single consumer) data gradient, each against plain fp32 PyTorch ops on
# identical inputs.  This covers EVERY parameter of the model element-wise, with the real plans / tile schedules.
def _nchw(t):
    return t.float().permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize("name,B,S", [("yolov4", 8, 640), ("yolov3", 4, 128)])
def test_train_step_layerwise(name, B, S):
    import torch.nn.functional as F
    from utils import utils as my_utils
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = attach_hyp(build_model(name, device="cuda")).train()
    model.use_cuda_graph = False
    x = orc.synth_images(B, S, S, seed=0).cuda()
    t = orc.synth_targets(B, 8, 80, seed=1).cuda()
    pred, _ = model(x)
    loss, items = my_utils.compute_loss(pred, t, model)
    loss.backward()
    torch.cuda.synchronize()
    plan = model.engine().last_plan
    consumers, sharers = {}, {}
    for r in plan.convs:
        if r.src is not None:
            consumers[id(r.src)] = consumers.get(id(r.src), 0) + 1
        if r.res is not None:                       # fused shortcut: dy also flows into the skip source
            consumers[id(r.res)] = consumers.get(id(r.res), 0) + 2
        for tt in (r.src, r.y):
            if tt is not None:
                sharers.setdefault(tt.buf.data_ptr(), set()).add(id(tt))
    for r in plan.convs:                            # tensors living inside a concat buffer receive gradient slices
        for tt in (r.src, r.y):                     # from the concat's consumer as well
            if tt is not None and (len(sharers[tt.buf.data_ptr()]) > 1 or tt.buf.shape[3] != tt.C):
                consumers[id(tt)] = consumers.get(id(tt), 0) + 2
    for st in plan.order:
        if st[0] != 'conv':
            for tt in st[1:]:
                for q in (tt if isinstance(tt, (list, tuple)) else [tt]):
                    if hasattr(q, 'buf'):
                        consumers[id(q)] = consumers.get(id(q), 0) + 2      # any non-conv consumer disqualifies
    worst = {"conv_fwd": 0.0, "bn_fwd": 0.0, "bn_bwd_dz": 0.0, "bn_dgamma": 0.0, "bn_dbeta": 0.0, "wgrad": 0.0,
             "dgrad": 0.0}
    n_dgrad = 0
    for r in plan.convs:
        conv, bn = r.conv, r.bn
        if r.stem or bn is None:
            continue
        w16 = conv.weight.detach().half().float()
        xin = _nchw(r.src.view())
        # conv forward on identical fp16 operands, fp32 accumulation
        z_ref = F.conv2d(xin, w16, None, conv.stride, conv.padding)
        z = _nchw(r.z.view())
        worst["conv_fwd"] = max(worst["conv_fwd"], float((z - z_ref).abs().max() / z_ref.pow(2).mean().sqrt()))
        # BatchNorm forward + activation (+ fused shortcut) from the engine's own z and the engine's own batch statistics
        # (taken on the fp32 accumulators in the conv epilogue; recomputing them from the fp16-rounded z moves them by
        # ~1e-4 sigma, which flips the leaky-ReLU branch of the few elements with |u| below that and would dominate a
        # max-norm comparison of the backward)
        mean_e, invstd_e = r.save[0].view(1, -1, 1, 1), r.save[1].view(1, -1, 1, 1)
        mean_r = z.mean(dim=(0, 2, 3)).view(1, -1, 1, 1)
        std_r = z.var(dim=(0, 2, 3), unbiased=False).add(bn.eps).sqrt().view(1, -1, 1, 1)
        worst["bn_stats"] = max(worst.get("bn_stats", 0.0), float(((mean_e - mean_r).abs() / std_r).max()),
                                float((invstd_e * std_r - 1).abs().max()))
        gam, bet = bn.weight.detach().float().view(1, -1, 1, 1), bn.bias.detach().float().view(1, -1, 1, 1)
        xhat = (z - mean_e) * invstd_e
        u = (xhat * gam + bet).requires_grad_(True)
        yr = orc.activation(u, r.act, r.slope)
        y_ref = yr.detach() + _nchw(r.res.view()) if r.res is not None else yr.detach()
        y = _nchw(r.y.view())
        worst["bn_fwd"] = max(worst["bn_fwd"], float((y - y_ref).abs().max() / y_ref.abs().max()))
        # BatchNorm backward from the engine's own dy
        dy = _nchw(plan.grad_of[id(r.y)].view())
        du, = torch.autograd.grad(yr, u, dy)
        N = z.shape[0] * z.shape[2] * z.shape[3]
        dbeta_ref = du.sum(dim=(0, 2, 3))
        dgamma_ref = (du * xhat).sum(dim=(0, 2, 3))
        ref_dz = gam * invstd_e * (du - dbeta_ref.view(1, -1, 1, 1) / N - xhat * dgamma_ref.view(1, -1, 1, 1) / N)
        aux = plan.dz_aux[r.aux_row]
        dz = _nchw(plan.dz_bufs[r.i]) * float(aux[2])
        safe = (u.detach().abs() > 1e-5).float()        # elements whose activation branch is not decided by fp32 rounding
        worst["bn_bwd_dz"] = max(worst["bn_bwd_dz"], float(((dz - ref_dz) * safe).abs().max() / ref_dz.abs().max().clamp(min=1e-30)))
        # Elements sitting on the kink of a piecewise-linear activation (|u| below fp32 rounding: the engine forms
        # u = fma(z, gamma*invstd, beta - mean*gamma*invstd), this reference ((z - mean)*invstd)*gamma + beta) take the
        # other branch in one of the two computations; ONE such element moves a channel's dbeta by up to |dy| -- 1e-2 of
        # the layer maximum on the 20x20 / 40x40 maps -- and which elements they are changes from run to run with the
        # summation order of the batch statistics (atomics).  Their worst-case contribution is therefore subtracted per
        # channel before the comparison (measured with tools/flake_probe.py: leaky layers only, 1e-3..3e-2 in ~1/3 of
        # the runs, never on the smooth Mish layers); everything else must agree to fp32 summation order.
        amb = (u.detach().abs() <= 1e-5).float()
        slack_b = (amb * dy.abs()).sum(dim=(0, 2, 3))
        slack_g = (amb * (dy * xhat).abs()).sum(dim=(0, 2, 3))
        e_g = float(((bn.weight.grad - dgamma_ref).abs() - slack_g).clamp(min=0).max() / dgamma_ref.abs().max())
        e_b = float(((bn.bias.grad - dbeta_ref).abs() - slack_b).clamp(min=0).max() / dbeta_ref.abs().max())
        if e_b > 1e-4 or e_g > 1e-4:        # diagnostics: which layer, how large its gradients are
            ch = int((bn.bias.grad - dbeta_ref).abs().argmax())
            print("  [layer %d %s out %dx%dx%d act=%s res=%s, %d elements on the kink] dgamma err %.3g (max |dgamma| %.3g) dbeta err %.3g (max |dbeta| "
                  "%.3g; channel %d: engine %.6g ref %.6g) max |dy| %.3g"
                  % (r.i, tuple(conv.weight.shape), z.shape[1], z.shape[2], z.shape[3], r.act, r.res is not None,
                     int(amb.sum()), e_g,
                     float(dgamma_ref.abs().max()), e_b, float(dbeta_ref.abs().max()), ch, float(bn.bias.grad[ch]),
                     float(dbeta_ref[ch]), float(dy.abs().max())))
        worst["bn_dgamma"] = max(worst["bn_dgamma"], e_g)
        worst["bn_dbeta"] = max(worst["bn_dbeta"], e_b)
        # weight gradient from the engine's own (x, dz)
        dw_ref = torch.nn.grad.conv2d_weight(xin, conv.weight.shape, dz, conv.stride, conv.padding)
        worst["wgrad"] = max(worst["wgrad"], float((conv.weight.grad - dw_ref).norm() / dw_ref.norm()))
        # data gradient where this conv is the only consumer of its input
        if consumers.get(id(r.src), 0) == 1 and id(r.src) in plan.grad_of:
            dx_ref = torch.nn.grad.conv2d_input(xin.shape, w16, dz, conv.stride, conv.padding)
            dx = _nchw(plan.grad_of[id(r.src)].view())
            worst["dgrad"] = max(worst["dgrad"], float((dx - dx_ref).abs().max() / dx_ref.abs().max()))
            n_dgrad += 1
        del z_ref, u, yr, y_ref, dy, dz, ref_dz, dw_ref, xin, du, xhat
    print("\n[%s train %dx%dx%d, layer-wise on the engine's own tensors] worst over %d BN conv layers (%d data-gradient "
          "checks): %s" % (name, B, S, S, sum(1 for r in plan.convs if r.bn is not None and not r.stem), n_dgrad,
                           " ".join("%s=%.3g" % kv for kv in worst.items())))
    assert n_dgrad >= 10
    assert worst["conv_fwd"] < 4e-3          # fp16 store of z: 2^-11 relative to the largest values, vs the rms
    assert worst["bn_stats"] < 2e-3          # epilogue statistics (fp32 accumulators) vs statistics of the stored fp16 z
    assert worst["bn_fwd"] < 2e-3            # fp16 store of y
    assert worst["bn_bwd_dz"] < 4e-3         # fp16 store of dz (power-of-two scaled)
    assert worst["bn_dgamma"] < 2e-3 and worst["bn_dbeta"] < 2e-3
    assert worst["wgrad"] < 2e-3             # fp32 accumulation order (split-K atomics)
    assert worst["dgrad"] < 1.6e-2           # bf16 store of the activation gradient (2^-8)
