"""GPU, world_size 2, NCCL: the data-parallel training path on real devices (b200yolo/parallel.py + train_engine.py).

Semantics under test (reference train.py:219-221 = DistributedDataParallel; SURVEY.md section 8e):
  * the reduced gradient is the MEAN over ranks of the per-rank gradients (each rank: its own image shard, its own
    batch-statistics BatchNorm, its own loss normalisation),
  * parameters are identical on both ranks after the fused SGD step,
  * BatchNorm running buffers follow rank 0 (broadcast_buffers) on the next forward.
The per-rank gradients are recomputed on rank 0 by the same engine WITHOUT the data-parallel wrapper (plain autograd
.grad path), so the comparison isolates the exchange step; the engine's gradients themselves are gated against the
oracle in tests/test_gpu_train_model.py.  Skipped when fewer than two GPUs are visible."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import helpers
from helpers import attach_hyp, build_model, orc

pytestmark = pytest.mark.gpu

NAME, SIZE, BATCH = "yolov3-tiny", 128, 4


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _shard(rank):
    x = orc.synth_images(BATCH, SIZE, SIZE, seed=10 + rank)
    t = orc.synth_targets(BATCH, 6, 80, seed=20 + rank)
    return x, t


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from b200yolo.parallel import FlatDataParallel
    from utils import utils as my_utils
    res = {}
    # per-rank reference gradients on rank 0: plain model, no wrapper, one shard at a time
    if rank == 0:
        ref = {}
        for r in range(world):
            m = attach_hyp(build_model(NAME, device=dev)).train()
            m.use_cuda_graph = False
            x, t = _shard(r)
            pred, _ = m(x.to(dev))
            loss, _ = my_utils.compute_loss(pred, t.to(dev), m)
            loss.backward()
            ref[r] = {k: p.grad.detach().float().cpu().clone() for k, p in m.named_parameters()}
            if r == 0:
                res["rank0_running_mean"] = m.module_list[0][1].running_mean.detach().cpu().clone()
        res["ref"] = ref
    model = attach_hyp(build_model(NAME, seed=rank, device=dev)).train()    # rank 1 starts from other weights
    dp = FlatDataParallel(model)                                            # ... and gets rank 0's at construction
    x, t = _shard(rank)
    x, t = x.to(dev), t.to(dev)
    for it in range(3):                       # eager, graph capture, graph replay
        dp.zero_grad()
        pred, _ = dp(x)
        loss, items = my_utils.compute_loss(pred, t, dp)
        loss.backward()
        if it == 0:
            res["local_norm"] = float(dp.flat_grad.norm())
            res["local"] = dp.flat_grad.detach().cpu().clone()
            dp.reduce_gradients()
            res["reduced"] = dp.flat_grad.detach().cpu().clone()
            res["avg"] = {n: dp.grad_views[id(p)].detach().cpu().clone() / world for n, p in zip(dp.names, dp.params)}
            res["running_mean_after_fwd"] = model.module_list[0][1].running_mean.detach().cpu().clone()
        else:
            dp.reduce_gradients()
        dp.step(lr=1e-3, momentum=0.937, weight_decay=0.000484)
    torch.cuda.synchronize()
    res["params"] = dp.flat_param.detach().cpu().clone()
    res["loss"] = float(loss)
    # buffers follow rank 0 on the next forward (N3)
    dp._broadcast_buffers()
    res["rm_synced"] = model.module_list[0][1].running_mean.detach().cpu().clone()
    out[rank] = res
    dist.destroy_process_group()


def test_two_rank_nccl_training_step():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    r0, r1 = out[0], out[1]
    # one all-reduce == mean of the per-rank gradients; both ranks hold the same reduced buffer
    worst, table = 0.0, []
    for k, g0 in r0["avg"].items():
        assert torch.equal(g0, r1["avg"][k]), k
        expect = (r0["ref"][0][k] + r0["ref"][1][k]) / 2
        err = float((g0 - expect).norm() / (expect.norm() + 1e-12))
        table.append((err, k, float(expect.norm()), float(g0.norm()), float(r0["ref"][0][k].norm()), float(r0["ref"][1][k].norm())))
        worst = max(worst, err)
    table.sort(reverse=True)
    print("\n[2-rank NCCL] reduced gradient vs mean of per-rank gradients recomputed without the wrapper: worst relative "
          "norm error %.3g (run-to-run noise of this ill-conditioned toy problem is of the same size, "
          "tests/test_gpu_train_model.py::test_flat_sink_matches_plain_autograd)" % worst)
    # the exchange step itself, exactly: the buffer after the ONE all-reduce is the sum of the two ranks' local buffers
    # (fp32 addition of two numbers is order independent -> bit exact), identical on both ranks
    assert torch.equal(r0["reduced"], r1["reduced"])
    assert torch.equal(r0["reduced"], r0["local"] + r1["local"])
    # and the local buffers are the per-rank gradients: same norms as the wrapper-free recomputation
    for k, g0 in list(r0["avg"].items())[:8]:
        exp = (r0["ref"][0][k] + r0["ref"][1][k]) / 2
        assert abs(float(g0.norm()) - float(exp.norm())) < 0.05 * float(exp.norm()), k
    # the ranks saw different shards
    assert abs(r0["local_norm"] - r1["local_norm"]) > 1e-6 * r0["local_norm"]
    # identical parameters after three fused optimiser steps (rank 1 started from a different seed)
    assert torch.equal(r0["params"], r1["params"])
    assert torch.isfinite(r0["params"]).all() and r0["loss"] == r0["loss"]
    # rank-0 running statistics win
    assert torch.equal(r0["rm_synced"], r1["rm_synced"])
    assert not torch.equal(r0["running_mean_after_fwd"], r1["running_mean_after_fwd"])
    assert torch.allclose(r0["running_mean_after_fwd"], r0["rank0_running_mean"], rtol=1e-3, atol=1e-5)
