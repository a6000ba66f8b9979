"""GPU: the grouped optimiser over FlatDataParallel's flat buffers (b200yolo/optim.py, csrc/train.cu opt_grouped_kernel)
against dp.step and against torch.optim built by train.py's code (train.py:120-144, burn-in :356-365, LambdaLR :201).
Gate: rtol 1e-5 / atol 1e-6 (the gate of tests/test_gpu_train_kernels.py::test_sgd_grouped_matches_torch); each test
prints its largest observed error."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from helpers import attach_hyp, build_model, cfg_path, orc
from optim_ref import HYP, burn_in, cosine_lf, torch_optimizer

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-5, 1e-6


def _model(name, quantized=-1, seed=0):
    if quantized == -1:
        return build_model(name, seed=seed, device="cuda")
    import models
    torch.manual_seed(seed)
    m = models.Darknet(cfg_path(name), quantized=quantized, a_bit=8, w_bit=8, shortcut_way=1, steps=100)
    return m.cuda()


def _pair(name, quantized=-1):
    """A FlatDataParallel model and a plain twin with the same parameters (the twin is what torch.optim updates)."""
    from b200yolo.parallel import FlatDataParallel
    dp = FlatDataParallel(_model(name, quantized))
    twin = _model(name, quantized, seed=1)
    src = dict(dp.module.named_parameters())
    with torch.no_grad():
        for n, p in twin.named_parameters():
            p.copy_(src[n])
    return dp, twin


def _feed(dp, twin, gen, scale=1e-2):
    """The same random gradient into the flat buffer (through the .grad views) and into the twin's .grad."""
    tp = dict(twin.named_parameters())
    for n, p in dp.module.named_parameters():
        g = (torch.randn(p.shape, generator=gen) * scale).cuda()
        p.grad.copy_(g)
        tp[n].grad = g.clone()


def _compare(dp, twin, opt, ref, keys, what):
    """Parameters and every state tensor of the flat optimiser against the torch one, within the gate; prints and
    returns the largest absolute difference."""
    tp = dict(twin.named_parameters())
    worst = 0.0
    for n, p in dp.module.named_parameters():
        q = tp[n]
        pairs = [(p.detach(), q.detach())] + [(opt.state[p][k], ref.state[q][k]) for k in keys]
        for a, b in pairs:
            worst = max(worst, float((a - b).abs().max()))
            np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=RTOL, atol=ATOL,
                                       err_msg="%s %s" % (what, n))
    print("\n[%s] max abs error over parameters and %s: %.3g" % (what, "/".join(keys), worst))
    return worst


def test_flat_sgd_bit_identical_to_dp_step():
    """Uniform hyper-parameters (one lr and momentum, weight decay on pg1 only, as dp.step): FlatSGD and dp.step run the
    same per-element expression, with the EMA and the BatchNorm-L1 term on, for 5 steps."""
    from b200yolo.optim import make_optimizer
    from b200yolo.parallel import FlatDataParallel
    dps = [FlatDataParallel(_model("yolov3-tiny")) for _ in range(2)]
    idx = [0, 2, 4, 6]
    for dp in dps:
        dp.enable_ema()
        dp.set_bn_sparsity(idx, 1e-3)
    hyp = dict(HYP, lr0=0.01)
    opt = make_optimizer(dps[1], hyp)
    gen = torch.Generator().manual_seed(5)
    start = dps[0].flat_param.clone()
    for _ in range(5):
        g = (torch.randn(dps[0].flat_grad.numel(), generator=gen) * 1e-2).cuda()
        for dp in dps:
            dp.flat_grad.copy_(g)
        dps[0].step(lr=hyp['lr0'], momentum=hyp['momentum'], weight_decay=hyp['weight_decay'])
        opt.step()
    torch.cuda.synchronize()
    a, b = dps
    moved = float((a.flat_param - start).abs().max())
    print("\n[FlatSGD vs dp.step] max |dp| moved %.3g, max |diff| param %.3g mom %.3g ema %.3g"
          % (moved, float((a.flat_param - b.flat_param).abs().max()), float((a.flat_mom - b.flat_mom).abs().max()),
             float((a.ema_param - b.ema_param).abs().max())))
    assert moved > 0
    assert torch.equal(a.flat_param, b.flat_param)
    assert torch.equal(a.flat_mom, b.flat_mom)
    assert torch.equal(a.ema_param, b.ema_param)
    assert torch.equal(a.ema_buf, b.ema_buf)


def test_flat_sgd_continues_the_momentum_of_dp_step():
    """One dp.step() and then two steps of make_optimizer's FlatSGD (uniform hyper-parameters) on the same dp: the
    FlatSGD continues the momentum dp.step left in flat_mom, bit for bit as three dp.step() calls."""
    from b200yolo.optim import make_optimizer
    from b200yolo.parallel import FlatDataParallel
    dps = [FlatDataParallel(_model("yolov3-tiny")) for _ in range(2)]
    hyp = dict(HYP, lr0=0.01)
    gen = torch.Generator().manual_seed(9)
    for i in range(3):
        g = (torch.randn(dps[0].flat_grad.numel(), generator=gen) * 1e-2).cuda()
        for dp in dps:
            dp.flat_grad.copy_(g)
        dps[0].step(lr=hyp['lr0'], momentum=hyp['momentum'], weight_decay=hyp['weight_decay'])
        if i == 0:
            dps[1].step(lr=hyp['lr0'], momentum=hyp['momentum'], weight_decay=hyp['weight_decay'])
            opt = make_optimizer(dps[1], hyp)
        else:
            opt.step()
    torch.cuda.synchronize()
    a, b = dps
    print("\n[dp.step then FlatSGD vs dp.step] max |diff| param %.3g mom %.3g"
          % (float((a.flat_param - b.flat_param).abs().max()), float((a.flat_mom - b.flat_mom).abs().max())))
    assert torch.equal(a.flat_param, b.flat_param)
    assert torch.equal(a.flat_mom, b.flat_mom)


def test_flat_sgd_burn_in_and_lambda_lr_match_torch_sgd():
    """train.py's burn-in (n_burn = 6, 4 batches per epoch) over 10 iterations, LambdaLR stepped at each epoch end."""
    from b200yolo.optim import make_optimizer
    dp, twin = _pair("yolov3-tiny")
    opt = make_optimizer(dp, HYP)
    ref = torch_optimizer(twin, HYP)
    epochs, nb, n_burn = 3, 4, 6
    lf = cosine_lf(epochs)
    scheds = [torch.optim.lr_scheduler.LambdaLR(o, lr_lambda=lf) for o in (opt, ref)]
    gen = torch.Generator().manual_seed(6)
    bias_lr_differs = False
    for ni in range(10):
        epoch = ni // nb
        if ni <= n_burn:
            for o in (opt, ref):
                burn_in(o, ni, n_burn, epoch, lf)
        lrs = [g['lr'] for g in opt.param_groups]
        bias_lr_differs |= lrs[2] != lrs[0] and lrs[2] != lrs[1]
        _feed(dp, twin, gen)
        opt.step()
        ref.step()
        if ni % nb == nb - 1:
            for s in scheds:
                s.step()
    assert bias_lr_differs
    assert [g['lr'] for g in opt.param_groups] == [g['lr'] for g in ref.param_groups]
    _compare(dp, twin, opt, ref, ("momentum_buffer",), "burn-in SGD")


@pytest.mark.parametrize("quantized", [-1, 1, 2])
def test_flat_adam_matches_torch_adam(quantized):
    """20 steps of --adam on the float model, and of the google (quantized=1) and TPSQ (quantized=2) groups."""
    from b200yolo.optim import FlatAdam, make_optimizer
    dp, twin = _pair("yolov3-tiny", quantized)
    hyp = dict(HYP, lr0=0.2)                         # Adam lr = lr0 * 0.005 = 1e-3
    opt = make_optimizer(dp, hyp, adam=True, quantized=quantized)
    ref = torch_optimizer(twin, hyp, adam=True, quantized=quantized)
    assert isinstance(opt, FlatAdam) and len(opt.param_groups) == (4 if quantized == 2 else 3)
    gen = torch.Generator().manual_seed(7)
    for _ in range(20):
        _feed(dp, twin, gen, scale=1.0)
        opt.step()
        ref.step()
    _compare(dp, twin, opt, ref, ("exp_avg", "exp_avg_sq"), "Adam quantized=%d" % quantized)
    assert float(opt.state[dp.params[0]]['step']) == 20.0


@pytest.mark.parametrize("adam", [False, True])
def test_state_dict_interop_with_torch(adam):
    """3 steps with one optimiser, its state_dict into the other kind, 3 more steps with both: flat -> torch and
    torch -> flat."""
    from b200yolo.optim import make_optimizer
    keys = ("exp_avg", "exp_avg_sq") if adam else ("momentum_buffer",)
    hyp = dict(HYP, lr0=0.2) if adam else HYP
    gen = torch.Generator().manual_seed(8)
    for direction in ("flat->torch", "torch->flat"):
        dp, twin = _pair("yolov3-tiny")
        opt = make_optimizer(dp, hyp, adam=adam)
        ref = torch_optimizer(twin, hyp, adam=adam)
        first, second = (opt, ref) if direction == "flat->torch" else (ref, opt)
        for _ in range(3):
            _feed(dp, twin, gen)
            first.step()
        # the other side takes the first one's parameters and optimiser state, as from a checkpoint
        src, dst = (dp.module, twin) if first is opt else (twin, dp.module)
        sp = dict(src.named_parameters())
        with torch.no_grad():
            for n, p in dst.named_parameters():
                p.copy_(sp[n])
        second.load_state_dict(first.state_dict())
        for _ in range(3):
            _feed(dp, twin, gen)
            opt.step()
            ref.step()
        _compare(dp, twin, opt, ref, keys, "state_dict %s %s" % ("Adam" if adam else "SGD", direction))


def test_end_to_end_training_steps_during_burn_in():
    """yolov3-tiny at 128^2 through FlatDataParallel: forward -> compute_loss -> backward -> FlatSGD.step() during
    burn-in, against torch.optim.SGD fed the same flat gradients; .grad stays the flat view through zero_grad()."""
    from utils import utils as my_utils
    from b200yolo.optim import make_optimizer
    dp, twin = _pair("yolov3-tiny")
    attach_hyp(dp.module).train()
    opt = make_optimizer(dp, HYP)
    ref = torch_optimizer(twin, HYP)
    lf = cosine_lf(3)
    for o in (opt, ref):
        torch.optim.lr_scheduler.LambdaLR(o, lr_lambda=lf)
    x = orc.synth_images(4, 128, 128, seed=10).cuda()
    t = orc.synth_targets(4, 6, 80, seed=20).cuda()
    tp = dict(twin.named_parameters())
    losses = []
    for ni in range(4):
        opt.zero_grad()
        assert all(p.grad is dp.grad_views[id(p)] for p in dp.params)
        assert not dp.flat_grad.any()
        for o in (opt, ref):
            burn_in(o, ni, 6, 0, lf)
        pred, _ = dp(x)
        loss, _ = my_utils.compute_loss(pred, t, dp)
        loss.backward()
        dp.reduce_gradients()
        losses.append(float(loss))
        for n, p in dp.module.named_parameters():
            tp[n].grad = dp.grad_views[id(p)].detach().clone()
        opt.step()
        ref.step()
    assert all(np.isfinite(losses)) and losses[-1] != losses[0]
    _compare(dp, twin, opt, ref, ("momentum_buffer",), "end-to-end burn-in (losses %s)"
             % ", ".join("%.4f" % v for v in losses))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _adam_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from b200yolo.optim import make_optimizer
    from b200yolo.parallel import FlatDataParallel
    dp = FlatDataParallel(build_model("yolov3-tiny", seed=rank, device=dev))   # rank 0's parameters at construction
    opt = make_optimizer(dp, dict(HYP, lr0=0.2), adam=True)
    gen = torch.Generator().manual_seed(100 + rank)                            # each rank its own gradients
    start = dp.flat_param.cpu().clone()
    for _ in range(3):
        opt.zero_grad()
        dp.flat_grad.copy_(torch.randn(dp.flat_grad.numel(), generator=gen).to(dev))
        dp.reduce_gradients()
        opt.step()
    torch.cuda.synchronize()
    out[rank] = (start, dp.flat_param.cpu().clone())
    dist.destroy_process_group()


def test_two_rank_nccl_flat_adam():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    out = mp.Manager().dict()
    mp.spawn(_adam_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    (s0, p0), (s1, p1) = out[0], out[1]
    assert torch.equal(s0, s1)                          # rank 1 started from rank 0's parameters
    assert torch.equal(p0, p1) and torch.isfinite(p0).all()
    print("\n[2-rank FlatAdam] parameters moved by up to %.3g, identical on both ranks" % float((p0 - s0).abs().max()))
    assert not torch.equal(p0, s0)
