#!/usr/bin/env python
"""Per-shape timing of the forward and data-gradient convolutions of one training step, optionally against a second
build of the library (measurement tool, not part of the product path).

    python tools/time_conv_shapes.py [--model yolov4] [--batch 8] [--reps 20] [--rounds 5]
                                     [--other PATH/libb200yolo.so] [--out FILE.json]

Records the C-ABI calls of one eager training step (b200yolo.lib.RECORD) and keeps the implicit-GEMM forward
(`b2y_conv2d_fwd_stats`, `b2y_conv2d_fwd`) and data-gradient (`b2y_conv2d_bwd_data`) launches.  One recorded launch of
each distinct (entry point, shape) is captured `reps` times in a CUDA graph and timed with CUDA events.  With --other,
the same recorded arguments also go to a second build of the library (for example the parent commit's), and the two
builds are timed in alternation, `rounds` times per shape with the order flipped every round, so that clock and
neighbour drift fall on both alike.  Each row reports the median per launch; the totals weight every shape by how often
the step launches it.
"""
import argparse
import collections
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (puts the package on sys.path; model builders)
import torch  # noqa: E402

CALLS = ("b2y_conv2d_fwd_stats", "b2y_conv2d_fwd", "b2y_conv2d_bwd_data")


def shape_of(args):
    d = args[0]._obj
    return "%dx%d s%d %d->%d in %dx%d out %dx%d" % (d.ksize, d.ksize, d.stride, d.in_c, d.out_c, d.in_h, d.in_w,
                                                   d.out_h, d.out_w)


def load_other(path):
    """A second copy of the library with the same prototypes as the in-tree one."""
    from b200yolo import lib
    other = ctypes.CDLL(os.path.abspath(path))
    for name in CALLS:
        res, argt = lib._PROTOS[name]
        fn = getattr(other, name)
        fn.restype = res
        fn.argtypes = argt
    return other


def graph_of(fn, args, reps):
    from b200yolo import lib
    a = args[:-1] + (lib.stream_ptr(),)             # the stream is the last argument of every entry point
    lib.check(fn(*a), "warm-up")                     # first use: function attributes, scratch buffers
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a = args[:-1] + (lib.stream_ptr(),)
        for _ in range(reps):
            fn(*a)
    g.replay()
    torch.cuda.synchronize()
    return g


def time_graph(g, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="yolov4")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--other", default="", help="a second libb200yolo.so to time against the in-tree build")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_conv_shapes.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    from b200yolo import lib
    from b200yolo.parallel import FlatDataParallel
    from utils import utils as my_utils
    model = bench.build_model(args.model, dev, 0, train=True)
    model.use_cuda_graph = False
    u8, tg = bench.synth_batch(args.batch, 100)
    x = (u8.to(dev).float() / 256.0).contiguous()
    t = tg.to(dev)
    dp = FlatDataParallel(model)

    def step():
        dp.zero_grad()
        pred, _ = dp(x)
        loss, _ = my_utils.compute_loss(pred, t, dp)
        loss.backward()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    calls = bench.record_calls(step)
    shapes = collections.OrderedDict()
    for name, a in calls:
        if name in CALLS:
            key = (name, shape_of(a))
            if key not in shapes:
                shapes[key] = {"n": 0, "args": a, "flops": bench.conv_desc_flops(name, a)}
            shapes[key]["n"] += 1
    builds = [("this", lib.raw())]
    if args.other:
        builds.append(("other", load_other(args.other)))
    rows = []
    for (name, shape), s in shapes.items():
        graphs = [(tag, graph_of(getattr(raw, name), s["args"], args.reps)) for tag, raw in builds]
        ms = {tag: [] for tag, _ in builds}
        for r in range(args.rounds):
            for tag, g in (graphs if r % 2 == 0 else graphs[::-1]):
                ms[tag].append(time_graph(g, args.reps))
        del graphs
        rows.append({"call": name, "shape": shape, "n": s["n"], "flops": s["flops"],
                     "ms": {tag: statistics.median(v) for tag, v in ms.items()},
                     "ms_all": ms})
    gpu = torch.cuda.get_device_name(0)
    print("%s, model=%s batch=%d, %d shapes, median of %d rounds of %d launches%s"
          % (gpu, args.model, args.batch, len(rows), args.rounds, args.reps,
             (", other = %s" % args.other) if args.other else ""))
    hdr = "%9s %9s %6s" % ("this ms", "other ms", "ratio") if args.other else "%9s" % "this ms"
    print("%s %4s %7s  %-22s %s" % (hdr, "n", "TF/s", "entry point", "shape"))
    tot = collections.defaultdict(float)
    for r in rows:
        a = r["ms"]["this"]
        tf = r["flops"] / a / 1e9 if a > 0 else 0.0
        tot[(r["call"], "this")] += r["n"] * a
        if args.other:
            b = r["ms"]["other"]
            tot[(r["call"], "other")] += r["n"] * b
            lead = "%9.4f %9.4f %6.3f" % (a, b, a / b)
        else:
            lead = "%9.4f" % a
        print("%s %4d %7.1f  %-22s %s" % (lead, r["n"], tf, r["call"], r["shape"]))
    print("--- per step (each shape times its launch count)")
    for name in CALLS:
        if (name, "this") in tot:
            if args.other:
                print("%9.3f %9.3f %6.3f  %s" % (tot[(name, "this")], tot[(name, "other")],
                                                 tot[(name, "this")] / tot[(name, "other")], name))
            else:
                print("%9.3f  %s" % (tot[(name, "this")], name))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "model": args.model, "batch": args.batch, "other": args.other,
                       "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
