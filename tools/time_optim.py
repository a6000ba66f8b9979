#!/usr/bin/env python
"""Cost of one optimiser step over yolov4's flat buffers (FlatDataParallel, 64.4 M parameters), timed with CUDA events:
  dp.step        -- FlatDataParallel.step: FlatSGD over two groups (decayed conv weights, the rest), one launch
  FlatSGD        -- b200yolo.optim, train.py's three groups, one launch
  FlatAdam       -- the same for Adam
  torch SGD/Adam -- torch.optim (foreach, its default on CUDA) over the same parameter views, train.py's groups
each with and without the fused EMA for the flat ones.  Every variant runs `--rounds` windows of `--reps` steps,
alternated, and reports the median ms per step and the HBM bytes of the flat kernels over that time against the
3.35 TB/s of the H100 SXM data sheet.

    python tools/time_optim.py [--reps 50] [--rounds 5]

Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM = 3.35e12
HYP = {'lr0': 0.01, 'momentum': 0.937, 'weight_decay': 0.0005}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    from helpers import build_model
    from optim_ref import torch_optimizer
    from b200yolo.optim import make_optimizer
    from b200yolo.parallel import FlatDataParallel
    dp = FlatDataParallel(build_model("yolov4", device="cuda"))
    n = dp.flat_param.numel()
    dp.flat_grad.normal_(0, 1e-3)
    sgd = make_optimizer(dp, HYP)
    adam = make_optimizer(dp, HYP, adam=True)
    t_sgd = torch_optimizer(dp.module, HYP)
    t_adam = torch_optimizer(dp.module, HYP, adam=True)

    def with_ema(fn):
        def run():
            dp.ema_param = ema
            fn()
            del dp.ema_param
        return run

    dp.enable_ema()
    ema = dp.ema_param
    del dp.ema_param
    dp.ema_buf = None                       # the running-statistics EMA is a separate axpby, not timed here
    variants = {
        "dp.step": (lambda: dp.step(lr=0.01), 20),
        "FlatSGD": (sgd.step, 20),
        "FlatAdam": (adam.step, 28),
        "dp.step+ema": (with_ema(lambda: dp.step(lr=0.01)), 28),
        "FlatSGD+ema": (with_ema(sgd.step), 28),
        "FlatAdam+ema": (with_ema(adam.step), 36),
        "torch.optim.SGD": (t_sgd.step, None),
        "torch.optim.Adam": (t_adam.step, None),
    }
    for fn, _ in variants.values():           # warm-up (and the first SGD step, which skips the momentum read)
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, (fn, _) in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                fn()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / args.reps)
    res = {"params": n, "gpu": torch.cuda.get_device_name(0)}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                             "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        pass
    for k, (_, bpp) in variants.items():
        ms = sorted(times[k])[len(times[k]) // 2]
        row = {"ms": round(ms, 4)}
        if bpp is not None:
            row["GB"] = round(bpp * n / 1e9, 3)
            row["GB/s"] = round(bpp * n / (ms * 1e-3) / 1e9, 1)
            row["of_3.35TB/s"] = round(bpp * n / (ms * 1e-3) / HBM, 3)
        res[k] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
