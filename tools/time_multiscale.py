#!/usr/bin/env python
"""Multi-scale training throughput: yolov4, 8 images per step, a new image size on every step.

train.py draws the size of each batch from 320 ... 640 in steps of 32 (`--img-size 320 640`, multi_scale on by default,
`random.randrange(10, 21) * 32`).  This tool follows that rule with a fixed seed on every step, so the engine sees 11
shapes in random order, as a user's default training run does.  Each step is forward, compute_loss, backward and a
FlatDataParallel optimiser step.  Every size is warmed up first (an eager step, then the captured graphs); the timed
window is at least 200 steps and ends in a device synchronise.

Printed (one JSON line): images/s, the plans built and CUDA graphs captured inside the timed window (counted by
wrapping the plan constructor and torch.cuda.CUDAGraph.capture_begin), memory_allocated / max_memory_allocated, and
the card's name and power limit.

    python tools/time_multiscale.py [--steps 200] [--batch 8] [--seed 0] [--root TREE]

--root selects the repository tree whose package is imported (default: the one this file lives in), so that two trees
can be timed with the same script.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="yolov4")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, os.path.join(root, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"))

    import tempfile
    import torch
    import models
    from b200yolo import cfggen, train_engine
    from b200yolo.parallel import FlatDataParallel
    from utils import utils as my_utils

    if not torch.cuda.is_available():
        raise SystemExit("time_multiscale.py needs a CUDA device (H100)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    counts = {"plans": 0, "graphs": 0}
    init = train_engine.TrainPlan.__init__
    capture = torch.cuda.CUDAGraph.capture_begin

    def counting_init(self, *a, **k):
        counts["plans"] += 1
        init(self, *a, **k)

    def counting_capture(self, *a, **k):
        counts["graphs"] += 1
        return capture(self, *a, **k)

    train_engine.TrainPlan.__init__ = counting_init
    torch.cuda.CUDAGraph.capture_begin = counting_capture

    torch.manual_seed(0)
    cfg_dir = tempfile.mkdtemp(prefix="b2y_ms_cfg_")
    m = models.Darknet(cfggen.write_cfg(args.model, cfg_dir), img_size=(640, 640)).to(dev)
    m.train()
    m.nc, m.gr = 80, 1.0
    m.hyp = {'giou': 3.54, 'cls': 37.4, 'cls_pw': 1.0, 'obj': 64.3, 'obj_pw': 1.0, 'iou_t': 0.20, 'fl_gamma': 0.0}
    dp = FlatDataParallel(m)
    B = args.batch
    g = torch.Generator().manual_seed(100)
    sizes = [32 * k for k in range(10, 21)]
    imgs = {S: (torch.randint(0, 256, (B, 3, S, S), dtype=torch.uint8, generator=g).float() / 256.0).to(dev)
            for S in sizes}
    nt = 8 * B
    t = torch.cat([torch.arange(B).repeat_interleave(8).float()[:, None],
                   torch.randint(0, 80, (nt, 1), generator=g).float(),
                   torch.rand(nt, 2, generator=g) * 0.9 + 0.05,
                   torch.exp(torch.rand(nt, 2, generator=g) * 3.4 - 3.9)], 1).to(dev)

    def step(S):
        dp.zero_grad()
        pred, _ = dp(imgs[S])
        loss, items = my_utils.compute_loss(pred, t, dp)
        (loss * (B / 64.0)).backward()
        dp.reduce_gradients()
        dp.step(lr=1e-4, momentum=0.937, weight_decay=0.000484)
        return items

    for S in sizes:                      # eager step, then the captured graphs, for every size
        step(S)
        step(S)
    torch.cuda.synchronize()
    rng = random.Random(args.seed)
    order = [rng.randrange(10, 21) * 32 for _ in range(args.steps)]
    before = dict(counts)
    t0 = time.perf_counter()
    for S in order:
        items = step(S)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0

    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # the figure is informative; the measurement stands without it
        power = "unavailable (%s)" % type(e).__name__
    print(json.dumps({
        "metric": "images/sec %s train, multi-scale 320-640 (train.py rule, seed %d)" % (args.model, args.seed),
        "value": B * args.steps / dt, "unit": "images/s", "steps": args.steps, "per_step_batch": B,
        "ms_per_step": 1e3 * dt / args.steps,
        "plans_built_timed": counts["plans"] - before["plans"],
        "graphs_captured_timed": counts["graphs"] - before["graphs"],
        "memory_allocated": torch.cuda.memory_allocated(dev),
        "max_memory_allocated": torch.cuda.max_memory_allocated(dev),
        "loss_items": [float(v) for v in items],
        "gpu": torch.cuda.get_device_name(dev), "power_limit": power, "tree": root}), flush=True)


if __name__ == "__main__":
    main()
