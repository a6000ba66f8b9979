"""Time every weight-gradient launch (b2y_conv2d_bwd_weight) of the yolov4 training step at 8 x 640 x 640 with CUDA
events: records the launches of one eager step, then replays each distinct shape `--reps` times inside a CUDA graph (no
host cost of the call in the window).  Prints one JSON line: per shape the launches per step, ms per launch, TF/s and
the kernel / split-K slices the host chooses, and the sum over the step.

    python tools/time_wgrad.py [--batch 8] [--reps 20]
"""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the package on sys.path; model builders)
import torch  # noqa: E402


def plan(d, sms):
    """(kernel, N tile width, split-K slices) that b2y_conv2d_bwd_weight chooses for descriptor d."""
    ksteps = -(-d.batch * d.out_h * d.out_w // 64)
    if d.ksize == 3 and d.in_c in (32, 64):
        bn = 64 if d.in_c == 32 else 32
        sp = min(max(1, sms // -(-d.out_c // bn)), ksteps)
        kern = "taps"
    else:
        cin = d.in_c
        bn = (128 if cin >= 128 else 64) if cin % 64 == 0 else (32 if cin % 32 == 0 else 16)
        if cin % 64 == 0 and cin % bn != 0 and cin > bn:
            bn = 64
        base = -(-d.out_c // 128) * -(-cin // bn) * d.ksize * d.ksize
        sp = max(1, min(-(-2 * sms // base), max(1, ksteps // 8)))
        kern = "general"
    per = -(-ksteps // sp)
    return kern, bn, -(-ksteps // per)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    from b200yolo import lib
    from b200yolo.parallel import FlatDataParallel
    from utils import utils as my_utils
    model = bench.build_model("yolov4", dev, 0, train=True)
    model.use_cuda_graph = False
    dp = FlatDataParallel(model)
    u8, tg = bench.synth_batch(args.batch, 100)
    x = (u8.to(dev).float() / 256.0).contiguous()
    t = tg.to(dev)

    def step():
        dp.zero_grad()
        pred, _ = dp(x)
        loss, _ = my_utils.compute_loss(pred, t, dp)
        loss.backward()

    for _ in range(2):
        step()
    calls = [(n, a) for n, a in bench.record_calls(step) if n == "b2y_conv2d_bwd_weight"]
    shapes = collections.OrderedDict()
    for n, a in calls:
        d = a[0]._obj
        key = (d.ksize, d.stride, d.in_c, d.out_c, d.in_h, d.in_w, d.out_h, d.out_w)
        shapes.setdefault(key, []).append(a)
    fn = getattr(lib.raw(), "b2y_conv2d_bwd_weight")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rows, total_ms, total_flops = [], 0.0, 0.0
    for key, arglist in shapes.items():
        a = arglist[0][:-1] + (lib.stream_ptr(),)
        fn(*a)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ac = a[:-1] + (lib.stream_ptr(),)           # the capture stream
            for _ in range(args.reps):
                fn(*ac)
        g.replay()
        torch.cuda.synchronize()
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        del g
        flops = bench.conv_desc_flops("b2y_conv2d_bwd_weight", a)
        kern, bn, splits = plan(a[0]._obj, sms)
        k, s, ci, co, h, w, ho, wo = key
        rows.append({"shape": "%dx%d s%d %d->%d in %dx%d out %dx%d" % (k, k, s, ci, co, h, w, ho, wo),
                     "n": len(arglist), "ms": ms, "tflops": flops / ms / 1e9, "kernel": kern, "block_n": bn,
                     "splits": splits})
        total_ms += ms * len(arglist)
        total_flops += flops * len(arglist)
    rows.sort(key=lambda r: -r["ms"] * r["n"])
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "batch": args.batch,
                      "launches_per_step": len(calls), "ms_per_step": total_ms,
                      "tflops": total_flops / total_ms / 1e9, "shapes": rows}))


if __name__ == "__main__":
    main()
