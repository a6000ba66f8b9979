"""CPU, world_size 2, gloo: host logic of the data-parallel path (b200yolo/parallel.py): parameter flattening,
rank-0 broadcast of parameters and BN buffers, the single gradient all-reduce and its mean-over-ranks semantics
(the same formula DDP(reference) produces, SURVEY.md section 4/8e)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import helpers  # noqa: F401  (sys.path)


def _real_model():
    """The real module tree (yolov3-tiny: conv blocks with BatchNorm, two bias-only head convs) on the CPU; the
    training plan's role -- writing per-rank gradients through model._b2y_grad_sink -- is played by the test."""
    import models
    return models.Darknet(helpers.cfg_path("yolov3-tiny"))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from b200yolo.parallel import FlatDataParallel, _is_decay_param
    torch.manual_seed(100 + rank)               # ranks start from different weights / buffers
    m = _real_model()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.01 * rank)
        m.module_list[0][1].running_mean.fill_(float(rank + 1))
    dp = FlatDataParallel(m)
    sink = m._b2y_grad_sink                      # what TrainPlan._emit / the wgrad unpack write into
    res = {}
    res["params"] = dp.flat_param.clone()
    res["names"] = list(dp.names)
    res["n_decay"] = dp.n_decay
    # params are views of the flat buffer
    dp.flat_param.mul_(1.0)
    res["views"] = all(p.data_ptr() >= dp.flat_param.data_ptr() for p in dp.params)
    # per-rank gradients written through the .grad views (what the training plan does through the sink)
    g = torch.Generator().manual_seed(7 + rank)
    local = []
    for p in dp.params:
        v = torch.randn(p.shape, generator=g)
        sink[id(p)].copy_(v)
        assert p.grad.data_ptr() == sink[id(p)].data_ptr()      # .grad IS the slice of the flat buffer
        local.append(v.reshape(-1))
    res["local_grad"] = torch.cat(local)
    dp.reduce_gradients()
    res["avg"] = dp.averaged_gradients().clone()
    # buffer broadcast: rank 0's running stats win
    m.train()
    dp._broadcast_buffers()
    res["rm"] = m.module_list[0][1].running_mean.clone()
    res["decay_flags"] = [_is_decay_param(n) for n in dp.names]
    out[rank] = res
    dist.destroy_process_group()


def test_flat_data_parallel_gloo():
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    r0, r1 = out[0], out[1]
    assert torch.equal(r0["params"], r1["params"]), "parameters must be broadcast from rank 0"
    assert r0["views"] and r1["views"]
    # one all-reduce == mean of the per-rank gradients, bit exact for 2 ranks
    expect = (r0["local_grad"] + r1["local_grad"]) / 2
    assert torch.equal(r0["avg"], expect) and torch.equal(r1["avg"], expect)
    assert torch.equal(r0["rm"], torch.ones(16)) and torch.equal(r1["rm"], torch.ones(16))
    # optimiser grouping of the reference: weight decay only on '...Conv2d.weight'
    names, flags = r0["names"], r0["decay_flags"]
    assert flags == [("Conv2d.weight" in n and ".bias" not in n) for n in names]
    import models
    ref = models.Darknet(helpers.cfg_path("yolov3-tiny"))
    n_decay = sum(p.numel() for n, p in ref.named_parameters() if "Conv2d.weight" in n)
    assert r0["n_decay"] == n_decay and names[0] == "module_list.0.Conv2d.weight"
    assert sorted(names) == sorted(n for n, _ in ref.named_parameters())
    assert r0["params"].numel() == sum(p.numel() for p in ref.parameters()) == 8852366


def test_bn_sparsity_range_table_points_at_the_bn_scales():
    """FlatDataParallel.set_bn_sparsity (BNOptimizer.updateBN, prune_utils.py:133-138): the host (offset, length) rows
    from which the optimiser's tile table flags the L1 term address exactly the BatchNorm scale vectors of the listed
    layers inside the flat buffers (the kernel itself is checked on the GPU, tests/test_gpu_train_kernels.py)."""
    from b200yolo.parallel import FlatDataParallel
    m = _real_model()
    dp = FlatDataParallel(m)
    prune_idx = [0, 4, 8, 12]
    dp.set_bn_sparsity(prune_idx, 0.001)
    table, s = dp._l1
    assert s == 0.001 and table.dtype == torch.int64 and tuple(table.shape) == (len(prune_idx), 2)
    for (off, ln), idx in zip(table.tolist(), prune_idx):
        bn = m.module_list[idx][1]
        assert isinstance(bn, nn.BatchNorm2d) and ln == bn.weight.numel()
        assert dp.flat_param[off:off + ln].data_ptr() == bn.weight.data_ptr()
        assert dp.flat_grad[off:off + ln].data_ptr() == bn.weight.grad.data_ptr()
    dp.set_bn_sparsity(prune_idx, 0.0)          # s = 0 switches it off
    assert dp._l1 is None
