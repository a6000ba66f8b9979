#!/usr/bin/env python
"""One quantisation-aware training step of yolov3-mobilenet: forward, compute_loss and backward at 416 x 416, batch 16,
the size train.py trains MobileNet at; --quantized 1 (google QAT, the default) or 2 (TPSQ).  The QAT graph is data
dependent (range trackers, freeze steps), so it runs eagerly, layer by layer; the step is timed with CUDA events after
--warmup steps.  Weights are the synthetic ones of the tests (every tensor whose name the float model shares).

Printed (one JSON line): ms per step, images/s, and the card's name and power limit.

    python tools/time_qat_mobilenet.py [--quantized 1] [--steps 5] [--warmup 2] [--batch 16] [--size 416]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"), ROOT,
                os.path.join(ROOT, "tests")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=416)
    ap.add_argument("--quantized", type=int, choices=(1, 2), default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_qat_mobilenet.py needs a CUDA device")
    import models
    from helpers import attach_hyp, cfg_path, orc
    from utils import utils as my_utils
    m = models.Darknet(cfg_path("yolov3-mobilenet"))
    sd = orc.synth_state_dict(m.state_dict(), 0)
    qm = models.Darknet(cfg_path("yolov3-mobilenet"), quantized=args.quantized, a_bit=8, w_bit=8, shortcut_way=1,
                        steps=100)
    qm.load_state_dict({k: sd.get(k, v) for k, v in qm.state_dict().items()})
    qm = attach_hyp(qm.cuda()).train()
    x = orc.synth_images(args.batch, args.size, args.size, seed=0).cuda()
    t = orc.synth_targets(args.batch, 8, 80, seed=1).cuda()

    def step():
        qm.zero_grad(set_to_none=True)
        pred, _ = qm(x)
        loss, _ = my_utils.compute_loss(pred, t, qm)
        loss.backward()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.steps):
        step()
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / args.steps
    out = {"model": "yolov3-mobilenet", "quantized": args.quantized, "batch": args.batch, "size": args.size,
           "ms_per_step": round(ms, 2), "images_per_s": round(args.batch * 1000.0 / ms, 1),
           "device": torch.cuda.get_device_name(0)}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
