"""Device-timed inference step (CUDA-graph replay of the fused forward):
   python tools/time_infer.py --model yolov3 --batch 32"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (model construction + synthetic batch helpers)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="yolov3")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    model = bench.build_model(args.model, dev, 0, train=False)
    model.static_outputs = True
    u8, _ = bench.synth_batch(args.batch, 200)
    x = (u8.to(dev).float() / 256.0).contiguous()
    with torch.no_grad():
        for _ in range(5):
            model(x)
        torch.cuda.synchronize()
        best = 1e9
        for rep in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                model(x)
            e1.record()
            torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) / args.steps)
    sw = {k: v for k, v in os.environ.items() if k.startswith("B2Y_")}
    print("%s bs%d: %.3f ms/step  %s" % (args.model, args.batch, best, sw))


if __name__ == "__main__":
    main()
