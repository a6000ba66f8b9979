#!/usr/bin/env python
"""Per-launch timing of one step of the H100 engine (measurement tool, not part of the product path).

    python tools/profile_calls.py --mode train|infer [--model yolov4] [--batch 8] [--size 640] [--out FILE.json]

Records every C-ABI call of ONE eager step (b200yolo.lib.RECORD), then replays each call `reps` times back to back and
times it with CUDA events (L2-warm: consecutive replays of a call re-use its operands).  Conv calls carry their
algorithmic FLOPs (2 M N K from the descriptor) -> TFLOP/s per layer; the table is aggregated by (entry point, shape).
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


def describe(name, args):
    from b200yolo.lib import ConvDesc
    a0 = args[0]
    d = getattr(a0, "_obj", None)
    if isinstance(d, ConvDesc):
        return "%dx%d s%d %d->%d in %dx%d out %dx%d" % (d.ksize, d.ksize, d.stride, d.in_c, d.out_c, d.in_h, d.in_w,
                                                       d.out_h, d.out_w), bench.conv_desc_flops(name, args)
    ints = [str(a) for a in args if isinstance(a, int) and not isinstance(a, bool)][:6]
    return " ".join(ints), 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="train", choices=["train", "infer", "ptq"])
    ap.add_argument("--model", default="yolov4")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--out", default="")
    ap.add_argument("--top", type=int, default=60)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    from b200yolo import lib
    from utils import utils as my_utils
    B = args.batch or (8 if args.mode == "train" else 32)
    if args.mode == "ptq":
        # INT8 graph of the PTQ-calibrated yolov3 (fixture scales; timing does not depend on the values)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from test_gpu_ptq import _load_quantised_model
        model, _ = _load_quantised_model()
    else:
        model = bench.build_model(args.model, dev, 0, train=args.mode == "train")
    model.use_cuda_graph = False
    u8, tg = bench.synth_batch(B, 100)
    x = (u8.to(dev).float() / 256.0).contiguous()
    t = tg.to(dev)
    if args.mode == "train":
        from b200yolo.parallel import FlatDataParallel
        dp = FlatDataParallel(model)

        def step():
            dp.zero_grad()
            pred, _ = dp(x)
            loss, _ = my_utils.compute_loss(pred, t, dp)
            loss.backward()
            dp.reduce_gradients()
            dp.step(lr=1e-4)
    else:
        def step():
            with torch.no_grad():
                model(x)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    step()
    e1.record()
    torch.cuda.synchronize()
    eager_ms = e0.elapsed_time(e1)
    calls = bench.record_calls(step)
    raw = lib.raw()
    rows = []
    for name, a in calls:
        fn = getattr(raw, name)
        fn(*a)
        torch.cuda.synchronize()
        # `reps` launches captured in a CUDA graph: the replay excludes the CPU cost of the eager call (ctypes,
        # tensor-map encodes), which would otherwise floor every small kernel at ~10 us
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ac = a[:-1] + (lib.stream_ptr(),)           # the stream is the last argument of every entry point
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
        shape, flops = describe(name, a)
        rows.append({"call": name, "shape": shape, "ms": ms, "flops": flops})
    agg = collections.OrderedDict()
    for r in rows:
        k = (r["call"], r["shape"])
        a = agg.setdefault(k, {"n": 0, "ms": 0.0, "flops": 0.0})
        a["n"] += 1
        a["ms"] += r["ms"]
        a["flops"] += r["flops"]
    total = sum(r["ms"] for r in rows)
    by_call = collections.Counter()
    for r in rows:
        by_call[r["call"]] += r["ms"]
    print("mode=%s model=%s batch=%d: %d calls, sum of isolated call times %.3f ms (eager step %.3f ms)"
          % (args.mode, args.model, B, len(rows), total, eager_ms))
    print("--- by entry point")
    for k, v in by_call.most_common():
        print("%8.3f ms %5.1f%%  %s" % (v, 100 * v / total, k))
    print("--- top (entry point, shape)")
    for (c, s), a in sorted(agg.items(), key=lambda kv: -kv[1]["ms"])[:args.top]:
        tf = a["flops"] / a["ms"] / 1e9 if a["flops"] else 0.0
        print("%8.3f ms %5.1f%% x%-3d %7.1f TF/s  %-28s %s" % (a["ms"], 100 * a["ms"] / total, a["n"], tf, c, s))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"mode": args.mode, "model": args.model, "batch": B, "eager_ms": eager_ms, "rows": rows}, f)


if __name__ == "__main__":
    main()
