#!/usr/bin/env python
"""Adaptive BatchNorm recalibration throughput: the step EagleEye_*_prune.py runs for every candidate sub-network
(compact_model.train(); torch.no_grad(); forwards over a tenth of the training set), at EagleEye's defaults: 416 x 416
images, batch 16.

The candidates are the channel-pruned yolov3 and yolov3-tiny models of tests/golden/pruned_case.npz (their kept widths
and weights, run at 416 px).  Each is compared with the stock model's grad-enabled training forward (the forward of a
training step, autograd recording it) at the same size.  Both run as captured CUDA graphs after one eager call; the
timed window is at least --iters forwards and is measured with CUDA events.

Per candidate the set-up cost is reported too, since EagleEye builds a fresh compact model for every candidate: the
forward-only plan's build on its own, the first call of a fresh model (plan build, weight pack and the eager forward), and
the second call, which captures the graph, without one replay.

Printed (one JSON line): per model ms per batch and images/s of the recalibration forward and of the stock training
forward, the set-up times in ms, and the card's name and power limit.

    python tools/time_adabn.py [--iters 50] [--batch 16] [--size 416]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"), ROOT,
                os.path.join(ROOT, "tests")]


def _timed(fn, iters):
    import torch
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def _wall(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=416)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_adabn.py needs a CUDA device (H100)")
    torch.cuda.set_device(0)
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainPlan, TrainShared
    from helpers import build_model, orc
    from pruned_models import build_pruned

    B, S = args.batch, args.size
    x = orc.synth_images(B, S, S, seed=0).cuda()
    out = {"batch": B, "size": S, "iters": args.iters}
    for name in ("yolov3", "yolov3-tiny"):
        r = {}
        # set-up of one candidate: a fresh model, as EagleEye builds one per candidate
        model = build_pruned(name, device="cuda").train()
        dev = torch.device("cuda", 0)
        r["plan_build_ms"] = _wall(lambda: TrainPlan(model, tuple(x.shape), dev, False, SlotStore(dev),
                                                     TrainShared(dev), forward_only=True))
        model = build_pruned(name, device="cuda").train()
        with torch.no_grad():
            first = _wall(lambda: model(x))
            capture = _wall(lambda: model(x))
            replay = _wall(lambda: model(x))
            r["first_call_ms"] = first
            r["graph_capture_ms"] = capture - replay
            for _ in range(3):
                model(x)
            ms = _timed(lambda: model(x), args.iters)
        r["recalibration_ms_per_batch"], r["recalibration_images_per_s"] = ms, B * 1e3 / ms
        del model
        stock = build_model(name, device="cuda").train()
        for _ in range(3):
            stock(x)
        ms = _timed(lambda: stock(x), args.iters)
        r["stock_train_forward_ms_per_batch"], r["stock_train_forward_images_per_s"] = ms, B * 1e3 / ms
        del stock
        torch.cuda.empty_cache()
        out[name] = {k: round(v, 3) for k, v in r.items()}
    out["device"] = torch.cuda.get_device_name(0)
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
