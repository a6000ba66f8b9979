"""Time the weight gradient of the narrow 3x3 layers (Cin 32 / 64) of the yolov4 training step at 8 x 640 x 640 with
CUDA events.  B2Y_WGRAD_TAPS=0 selects the general kernel instead of the tap-transposed one (read once per process), so
compare two processes:

    python tools/time_wgrad.py; B2Y_WGRAD_TAPS=0 python tools/time_wgrad.py
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"))

# (batch, input H = W, Cin, Cout, stride) of the yolov4 layers the tap-transposed kernel serves
LAYERS = [(8, 640, 32, 64, 2), (8, 320, 64, 64, 1), (8, 320, 32, 64, 1), (8, 320, 64, 64, 1)]


def main():
    from b200yolo import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    out = {"gpu": torch.cuda.get_device_name(0), "taps": os.environ.get("B2Y_WGRAD_TAPS", "1") != "0", "layers": []}
    for B, S, ci, co, st in LAYERS:
        so = (S + 2 - 3) // st + 1
        x = torch.randn(B, S, S, ci, device="cuda", generator=g).half()
        dy = torch.randn(B, so, so, co, device="cuda", generator=g).half()
        dw = torch.zeros(co, 3, 3, ci, device="cuda")
        for _ in range(3):
            ops.conv2d_bwd_weight(x, dy, 3, st, 1, dw=dw)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for _ in range(n):
            ops.conv2d_bwd_weight(x, dy, 3, st, 1, dw=dw)
        e1.record()
        e1.synchronize()
        out["layers"].append({"shape": "B%d %dx%d %d->%d s%d" % (B, S, S, ci, co, st), "ms": e0.elapsed_time(e1) / n})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
