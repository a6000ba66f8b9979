#!/usr/bin/env python
"""Quantisation-aware training of yolov3-ghost at 416 x 416, batch 16 (the cfg's batch): the median time of one training
step (forward, compute_loss, backward) and of one eval forward over the steps of one run; --quantized 1 (google QAT,
the default, with --shortcut-way 1 or 2) or 2 (TPSQ).  The QAT graph is data dependent (range trackers, freeze steps),
so it runs eagerly, layer by layer, on the module forwards; each step is timed with CUDA events after --warmup steps.
Weights are the synthetic ones of the tests (every tensor whose name the float model shares).

Printed (one JSON line): median ms per training step and per eval forward, images/s of each, and the card's name and
power limit.

    python tools/time_qat_ghostnet.py [--quantized 1] [--shortcut-way 1] [--steps 10] [--warmup 2] [--batch 16]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"), ROOT,
                os.path.join(ROOT, "tests")]


def _median_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    events = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for start, end in events:
        start.record()
        fn()
        end.record()
    torch.cuda.synchronize()
    times = sorted(s.elapsed_time(e) for s, e in events)
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=416)
    ap.add_argument("--quantized", type=int, choices=(1, 2), default=1)
    ap.add_argument("--shortcut-way", type=int, choices=(1, 2), default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_qat_ghostnet.py needs a CUDA device")
    import models
    from helpers import attach_hyp, cfg_path, orc
    from utils import utils as my_utils
    m = models.Darknet(cfg_path("yolov3-ghost"))
    sd = orc.synth_state_dict(m.state_dict(), 0)
    qm = models.Darknet(cfg_path("yolov3-ghost"), quantized=args.quantized, a_bit=8, w_bit=8,
                        shortcut_way=args.shortcut_way, steps=100)
    qm.load_state_dict({k: sd.get(k, v) for k, v in qm.state_dict().items()})
    qm = attach_hyp(qm.cuda())
    x = orc.synth_images(args.batch, args.size, args.size, seed=0).cuda()
    t = orc.synth_targets(args.batch, 8, 80, seed=1).cuda()

    def train_step():
        qm.zero_grad(set_to_none=True)
        pred, _ = qm(x)
        loss, _ = my_utils.compute_loss(pred, t, qm)
        loss.backward()

    def eval_forward():
        with torch.no_grad():
            qm(x)

    qm.train()
    train_ms = _median_ms(train_step, args.steps, args.warmup)
    qm.eval()
    eval_ms = _median_ms(eval_forward, args.steps, args.warmup)
    out = {"model": "yolov3-ghost", "quantized": args.quantized, "shortcut_way": args.shortcut_way,
           "batch": args.batch, "size": args.size, "steps": args.steps,
           "train_ms_median": round(train_ms, 2), "train_images_per_s": round(args.batch * 1000.0 / train_ms, 1),
           "eval_ms_median": round(eval_ms, 2), "eval_images_per_s": round(args.batch * 1000.0 / eval_ms, 1),
           "device": torch.cuda.get_device_name(0)}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
