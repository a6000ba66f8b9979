#!/usr/bin/env python
"""INT8 PTQ inference throughput of the H100 engine (BASELINE configs[4]: yolov3.cfg, quantized=3 eval graph, int8 codes
with power-of-two scales, int8 wgmma convolutions).  The quantiser state is the one calibrated by the reference's
own PTQ flow (tests/golden/yolov3_64_ptq.npz); timing does not depend on the values.

    python tests/bench_ptq.py [--batch 32] [--size 640] [--steps 10]

Prints one JSON line.  Secondary benchmark: bench.py (the driver contract) measures configs[1].  Lives under tests/
because it builds the quantised model with the test helpers (synthetic weights from oracle/, fixture scales); the
timed region is the engine's INT8 graph only."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import helpers  # noqa: F401  (puts the package on sys.path)
    from test_gpu_ptq import _load_quantised_model
    qm, _ = _load_quantised_model()
    g = torch.Generator().manual_seed(0)
    x = (torch.randint(0, 256, (args.batch, 3, args.size, args.size), dtype=torch.uint8, generator=g).float() / 256.0).cuda()
    with torch.no_grad():
        for _ in range(args.warmup):
            qm(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            qm(x)
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    print(json.dumps({"metric": "images/sec (%dx%d) yolov3 INT8 PTQ inference" % (args.size, args.size),
                      "value": args.batch / (ms / 1e3), "unit": "images/s", "n_gpus": 1, "ms_per_step": ms,
                      "batch": args.batch, "dtype": "int8 codes / int32 accumulate", "data": "synthetic"}))


if __name__ == "__main__":
    main()
