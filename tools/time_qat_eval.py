#!/usr/bin/env python
"""One eval batch of a google-QAT (quantized=1) model, yolov3 and yolov3-tiny at 416 x 416, batch 32: on the captured
INT8 graph (b200yolo/qengine.py, what model.eval(); model(imgs) runs) and on the QAT module forwards it replaces
(b200yolo/qat.py QatRunner).  The QAT state comes from two training steps on the synthetic weights of the tests; the
two paths are checked to give the same outputs before anything is timed.  Each path runs --warmup batches, then --reps
timed windows of --iters batches (CUDA events); the median window is reported per batch, alternating the two paths.

Printed (one JSON line per model): median ms per batch of each path, the ratio, and the card's name and power limit.

    python tools/time_qat_eval.py [--batch 32] [--size 416] [--iters 10] [--reps 5] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"), ROOT,
                os.path.join(ROOT, "tests")]


def _model(name):
    import torch
    import models
    from helpers import attach_hyp, cfg_path, orc
    from utils import utils as my_utils
    sd = orc.synth_state_dict(models.Darknet(cfg_path(name)).state_dict(), 0)
    qm = models.Darknet(cfg_path(name), quantized=1, a_bit=8, w_bit=8, shortcut_way=1, steps=100)
    with torch.no_grad():
        for i, m in enumerate(qm.module_list):
            pre = 'module_list.%d.' % i
            if m.__class__.__name__ == 'Sequential' and len(m) and hasattr(m[0], 'activation_quantizer'):
                c = m[0]
                c.weight.copy_(sd[pre + 'Conv2d.weight'])
                if (pre + 'BatchNorm2d.weight') in sd:
                    c.gamma.copy_(sd[pre + 'BatchNorm2d.weight'])
                    c.beta.copy_(sd[pre + 'BatchNorm2d.bias'])
                else:
                    c.bias.copy_(sd[pre + 'Conv2d.bias'])
    qm = attach_hyp(qm.cuda()).train()
    for k in range(2):
        pred, _ = qm(orc.synth_images(2, 64, 64, seed=k).cuda())
        loss, _ = my_utils.compute_loss(pred, orc.synth_targets(2, 6, 80, seed=k + 1).cuda(), qm)
        loss.backward()
    return qm.eval()


def _window(fn, iters):
    import torch
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=416)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", default="yolov3,yolov3-tiny")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_qat_eval.py needs a CUDA device")
    from helpers import orc
    from b200yolo.qat import QatRunner
    from b200yolo.qengine import int8_graph_refusal
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    for name in args.models.split(","):
        qm = _model(name)
        assert int8_graph_refusal(qm) is None
        x = orc.synth_images(args.batch, args.size, args.size, seed=3).cuda()

        def int8():
            with torch.no_grad():
                return qm(x)

        def runner():
            with torch.no_grad():
                return QatRunner(qm).forward(x)

        a, b = int8(), runner()
        same = bool(torch.equal(a[0], b[0]))
        for _ in range(args.warmup):
            int8()
            runner()
        torch.cuda.synchronize()
        t8, tr = [], []
        for _ in range(args.reps):
            t8.append(_window(int8, args.iters))
            tr.append(_window(runner, args.iters))
        m8, mr = statistics.median(t8), statistics.median(tr)
        print(json.dumps({"model": name, "quantized": 1, "batch": args.batch, "size": args.size,
                          "int8_graph_ms": round(m8, 2), "qat_runner_ms": round(mr, 2), "speedup": round(mr / m8, 2),
                          "int8_graph_ms_all": [round(v, 2) for v in t8], "qat_runner_ms_all": [round(v, 2) for v in tr],
                          "outputs_equal": same, "device": torch.cuda.get_device_name(0), "power_limit": power}))


if __name__ == "__main__":
    main()
