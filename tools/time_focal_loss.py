#!/usr/bin/env python
"""Cost of the focal loss in the fused YOLO loss: b2y_yolo_loss (forward + d loss / d p) over the three yolov4 heads
of an 8 x 640^2 batch, at hyp['fl_gamma'] = 0 (plain BCE) and 1.5, timed with CUDA events, the two settings alternated.

    python tools/time_focal_loss.py [--batch 8] [--size 640] [--targets 20] [--reps 200] [--rounds 5]

Prints one JSON line: per-call milliseconds of all three heads for each gamma (median over rounds) and the GPU."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

# yolov4.cfg anchors (pixels) and their masks, strides 8 / 16 / 32
ANCHORS = [(12, 16), (19, 36), (40, 28), (36, 75), (76, 55), (72, 146), (142, 110), (192, 243), (459, 401)]
MASKS = [(0, 1, 2), (3, 4, 5), (6, 7, 8)]
STRIDES = [8, 16, 32]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--targets", type=int, default=20, help="targets per image")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    from b200yolo import ops
    from oracle import darknet_oracle as orc
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    heads = []
    for mask, s in zip(MASKS, STRIDES):
        n = args.size // s
        p = torch.randn(args.batch, 3, n, n, 85, generator=g).to(dev)
        av = torch.tensor([ANCHORS[a] for a in mask], dtype=torch.float32, device=dev) / s
        heads.append((p, av))
    t = orc.synth_targets(args.batch, args.targets, 80, seed=1).to(dev)
    hyp = orc.DEFAULT_HYP

    def step(gamma):
        for p, av in heads:
            ops.yolo_loss_layer(p, t, av, hyp['iou_t'], 1.0, hyp['cls_pw'], hyp['obj_pw'], hyp['giou'], hyp['obj'],
                                hyp['cls'], want_grad=True, fl_gamma=gamma)

    gammas = (0.0, 1.5)
    for gm in gammas:
        for _ in range(10):
            step(gm)
    torch.cuda.synchronize()
    times = {gm: [] for gm in gammas}
    for _ in range(args.rounds):
        for gm in gammas:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                step(gm)
            b.record()
            b.synchronize()
            times[gm].append(a.elapsed_time(b) / args.reps)
    med = {gm: sorted(v)[len(v) // 2] for gm, v in times.items()}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"workload": "b2y_yolo_loss fwd+bwd, yolov4 heads, %d x %d^2, %d targets"
                      % (args.batch, args.size, args.batch * args.targets),
                      "ms_gamma0": round(med[0.0], 4), "ms_gamma1.5": round(med[1.5], 4),
                      "ratio": round(med[1.5] / med[0.0], 3),
                      "rounds_gamma0": [round(v, 4) for v in times[0.0]],
                      "rounds_gamma1.5": [round(v, 4) for v in times[1.5]], "gpu": gpu}))


if __name__ == "__main__":
    main()
