#!/usr/bin/env python
"""INT8 PTQ inference throughput (BASELINE configs[4]: yolov3.cfg, quantized=3) with the WHOLE flow on the device and no
test infrastructure: PTQ.py's calibration (`q_model.train()` + forwards over calibration batches, b200yolo/qcalib.py:
cosine votes, bias correction, shortcut / concat searches) on two small synthetic batches, then the INT8 eval graph
(int8 wgmma convolutions, power-of-two requantisation) at the benchmark size.

    python tools/bench_ptq_native.py [--batch 32] [--size 640] [--steps 10]

Prints one JSON line.  bench.py runs this in a subprocess for its `secondary.yolov3_int8_ptq_infer_bs32` block."""
import argparse
import contextlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200")
sys.path.insert(0, PKG)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import models
    from b200yolo import cfggen
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    cfg = cfggen.write_cfg("yolov3", "/tmp/b2y_cfg_ptq_%d" % os.getpid())
    with contextlib.redirect_stdout(sys.stderr):
        qm = models.Darknet(cfg, img_size=(args.size, args.size), quantized=3, a_bit=8, w_bit=8, shortcut_way=1)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():          # non-degenerate BatchNorm statistics (the quantised conv owns gamma / beta / running_*)
        for m in qm.module_list:
            if m.__class__.__name__ == 'Sequential' and len(m) and hasattr(m[0], 'activation_quantizer'):
                c = m[0]
                if hasattr(c, 'running_var') and c.running_var is not None:
                    c.running_var.copy_(torch.rand(c.running_var.shape, generator=g) * 0.4 + 0.8)
                    c.running_mean.copy_(torch.randn(c.running_mean.shape, generator=g) * 0.1)
    qm = qm.cuda()
    qm.train()                     # PTQ.py:76-88: calibration forwards
    with torch.no_grad():
        for seed in (10, 11):
            gi = torch.Generator().manual_seed(seed)
            xc = (torch.randint(0, 256, (2, 3, 64, 64), dtype=torch.uint8, generator=gi).float() / 256.0).cuda()
            qm(xc)
    qm.eval()                      # PTQ.py:92-102: INT8 inference
    x = (torch.randint(0, 256, (args.batch, 3, args.size, args.size), dtype=torch.uint8, generator=g).float() / 256.0).cuda()
    with torch.no_grad():
        for _ in range(max(3, args.warmup)):
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
                      "batch": args.batch, "dtype": "int8 codes / int32 accumulate", "data": "synthetic",
                      "calibration": "native (b200yolo/qcalib.py), 2 batches of 2x64x64"}), flush=True)


if __name__ == "__main__":
    main()
