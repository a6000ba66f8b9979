#!/usr/bin/env python
"""N eager (or graph-replayed) YOLOv4 training steps, 8 images, 640x640 -- the bench.py headline workload without the
measurement scaffolding; a target for profiler captures.

    python tools/train_step.py [--steps 2] [--model yolov4] [--batch 8] [--graph]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--model", default="yolov4")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--graph", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    from b200yolo.parallel import FlatDataParallel
    from utils import utils as my_utils
    model = bench.build_model(args.model, dev, 0, train=True)
    model.use_cuda_graph = bool(args.graph)
    dp = FlatDataParallel(model)
    u8, tg = bench.synth_batch(args.batch, 100)
    x = (u8.to(dev).float() / 256.0).contiguous()
    t = tg.to(dev)
    for _ in range(args.steps):
        dp.zero_grad()
        pred, _ = dp(x)
        loss, items = my_utils.compute_loss(pred, t, dp)
        (loss * (args.batch / 64.0)).backward()
        dp.reduce_gradients()
        dp.step(lr=1e-4)
    torch.cuda.synchronize()
    print("loss items", [float(v) for v in items])


if __name__ == "__main__":
    main()
