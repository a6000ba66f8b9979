#!/usr/bin/env python
"""Training-step throughput of the H100 engine (BASELINE configs[2]: yolov4.cfg, 8 images / GPU, 640x640):
forward (batch-stat BN) + YOLO loss + backward + ONE gradient all-reduce + fused SGD-Nesterov.

    python tools/bench_train.py [--model yolov4] [--batch 8] [--size 640] [--steps 10]
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/bench_train.py ...

Prints one JSON line (rank 0).  Secondary benchmark: bench.py (the driver contract) measures configs[1]."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200")
sys.path.insert(0, PKG)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="yolov4")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", default="")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", init_method="env://", device_id=dev)
    import models
    from b200yolo import cfggen
    from b200yolo.parallel import FlatDataParallel
    from utils import utils as my_utils
    torch.manual_seed(0)
    m = models.Darknet(cfggen.write_cfg(args.model, "/tmp/b2y_cfg_train"), img_size=(args.size, args.size)).to(dev)
    m.train()
    m.nc, m.gr = 80, 1.0
    m.hyp = {'giou': 3.54, 'cls': 37.4, 'cls_pw': 1.0, 'obj': 64.3, 'obj_pw': 1.0, 'iou_t': 0.20, 'fl_gamma': 0.0}
    dp = FlatDataParallel(m)
    B = args.batch
    g = torch.Generator().manual_seed(100 + rank)
    x = (torch.randint(0, 256, (B, 3, args.size, args.size), dtype=torch.uint8, generator=g).float() / 256.0).to(dev)
    nt = 8 * B
    t = torch.cat([torch.arange(B).repeat_interleave(8).float()[:, None],
                   torch.randint(0, 80, (nt, 1), generator=g).float(),
                   torch.rand(nt, 2, generator=g) * 0.9 + 0.05,
                   torch.exp(torch.rand(nt, 2, generator=g) * 3.4 - 3.9)], 1).to(dev)

    def step():
        dp.zero_grad()
        pred, _ = dp(x)
        loss, items = my_utils.compute_loss(pred, t, dp)
        (loss * (B * world / 64.0)).backward()          # train.py:437 loss *= batch_size / 64
        dp.reduce_gradients()
        dp.step(lr=1e-4, momentum=0.937, weight_decay=0.000484)
        return items

    for _ in range(args.warmup):
        items = step()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        items = step()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / args.steps], device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(json.dumps({"metric": "images/sec (%dx%d) %s train" % (args.size, args.size, args.model),
                          "value": world * B / (float(ms) / 1e3), "unit": "images/s", "n_gpus": world,
                          "ms_per_step": float(ms), "per_gpu_batch": B, "loss_items": [float(v) for v in items],
                          "dtype": "f16 activations / bf16 gradients / f32 master", "data": "synthetic"}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
