#!/usr/bin/env python
"""bench.py -- images/sec of the Darknet hot path on H100 (BASELINE.json metric: "images/sec (640x640) YOLOv4
train+infer at 1/2/4/8 GPUs; conv roofline %").

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 ... bench.py --gpus N ...

PRIMARY workload (the headline `value`) = BASELINE.json configs[2], the per-GPU slice of "yolov4.cfg training bs=64 on
8 GPUs": yolov4.cfg, 8 images per GPU, 640x640, one process per GPU.  A "step" is one complete training step:

    forward (batch-statistics BatchNorm, wgmma convs) -> YOLO loss -> backward (dgrad / wgrad wgmma, BN backward)
    -> ONE NCCL all-reduce over the flat fp32 gradient buffer (N > 1) -> fused SGD-Nesterov

Per-GPU work is fixed as N grows ("scaling": "weak"; global batch = 8 N).  One JSON line on stdout (rank 0):
  value    : images/s, batch and targets resident in HBM (CUDA events around K steps, max over ranks)
  e2e      : the same step through the public API with pinned HOST uint8 images + targets: H2D copy, /256, step,
             D2H of the four loss items -- all inside the timed region
  roofline : the wgmma convolution family (forward, data gradient, weight gradient) of one step, replayed back to
             back and timed live with CUDA events; FLOPs = 2 M N K of every launch
  cpu_baseline : the oracle (CPU restatement of the reference's PyTorch path) training step on the host cores (N=1)
  secondary: (N=1) YOLOv3 inference bs 32 (configs[1]), YOLOv4 inference bs 32, with their own conv rooflines
--impl reference: the reference arm = the reference's own CPU PyTorch training step, restated in oracle/ and pinned to
the reference by tests/test_oracle_golden.py, all host threads, bounded sample.
--dump-outputs DIR: after the timed steps, write what the last timed training step computed (loss items, a fixed
sample of the three prediction tensors and of the flat gradient buffer) as DIR/<name>.npy; the inputs are seeded, so two
builds can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
import traceback

ROOT = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200")
sys.path.insert(0, PKG)

import torch  # noqa: E402

SIZE = 640
TRAIN_MODEL, TRAIN_BATCH = "yolov4", 8          # BASELINE configs[2]: bs 64 over 8 GPUs
INFER_BATCH = 32                                 # BASELINE configs[1]
# algorithmic conv FLOPs / image (BASELINE.md section 2, hooks on the reference's own modules)
FLOPS_FWD = {"yolov3": 155.89e9, "yolov4": 142.26e9}
FLOPS_TRAIN = {"yolov3": 467.7e9, "yolov4": 426.8e9}
HYP = {'giou': 3.54, 'cls': 37.4, 'cls_pw': 1.0, 'obj': 64.3, 'obj_pw': 1.0, 'iou_t': 0.20, 'fl_gamma': 0.0}
CONV_CALLS = ("b2y_conv2d_fwd", "b2y_conv2d_fwd_stats", "b2y_conv2d_bwd_data", "b2y_conv2d_bwd_weight")


def peaks():
    # NVIDIA's data sheet for the H100 SXM (700 W): dense FP16 / BF16 tensor rate and HBM3 bandwidth.  Denominators only:
    # a power-limited card runs below them.
    return {"hbm_gbs": 3350.0, "tflops": 989.0, "source": "H100 SXM data sheet (dense fp16, 700 W)"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index = index
        self.lines = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "200"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.proc.terminate()
        sm, mx, reasons = [], 0, set()
        for ln in self.lines:
            f = [c.strip() for c in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx = max(mx, float(f[1]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons),
                "samples": len(sm)}


def cfg_for(name, rank=0):
    """Generated cfg in a per-process directory (several ranks never write the same file; write_cfg renames atomically)."""
    from b200yolo import cfggen
    d = os.path.join("/tmp", "b2y_cfg_%d_r%d" % (os.getpid(), rank))
    return cfggen.write_cfg(name, d)


def build_model(name, device, rank=0, train=False):
    import contextlib
    import models
    torch.manual_seed(0)
    with contextlib.redirect_stdout(sys.stderr):       # "Model Summary: ..." must not pollute the one-JSON-line stdout
        m = models.Darknet(cfg_for(name, rank), img_size=(SIZE, SIZE))
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():  # non-degenerate BN statistics for eval (SURVEY.md section 8d)
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) * 0.4 + 0.8)
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
    m = m.to(device)
    if train:
        m.train()
        m.nc, m.gr, m.hyp = 80, 1.0, dict(HYP)
    else:
        m.eval()
        m.static_outputs = True   # return the engine's output buffers (no per-step clone)
    return m


def synth_batch(batch, seed):
    """uint8 images + [nT, 6] targets of SURVEY.md section 8d (8 boxes per image)."""
    g = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, (batch, 3, SIZE, SIZE), dtype=torch.uint8, generator=g)
    nt = 8 * batch
    t = torch.cat([torch.arange(batch).repeat_interleave(8).float()[:, None],
                   torch.randint(0, 80, (nt, 1), generator=g).float(),
                   torch.rand(nt, 2, generator=g) * 0.9 + 0.05,
                   torch.exp(torch.rand(nt, 2, generator=g) * 3.4 - 3.9)], 1)
    return u8, t


def host_threads():
    try:
        avail = len(os.sched_getaffinity(0))      # cores this process may be scheduled on
    except AttributeError:
        avail = os.cpu_count()
    try:                                           # ... and the cgroup CPU quota, if any (cpu.max = "<quota> <period>")
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            avail = max(1, min(avail, int(float(q) / float(per) + 0.5)))
    except (OSError, ValueError):
        pass
    return avail


# ----------------------------------------------------------------------------------------------------------------
# CPU arm: the reference's PyTorch path restated in oracle/ (test infrastructure; only timed here, never shipped)
# ----------------------------------------------------------------------------------------------------------------
def cpu_reference_rate(kind, name, max_seconds=20.0, batch=2, max_iters=10, threads=None):
    """kind = 'train' (forward + compute_loss + backward) or 'infer' (eval forward) of `name` at 640x640 on the host
    cores; bounded sample.  Returns the cpu_baseline dict (+ ms_per_step)."""
    sys.path.insert(0, ROOT)
    import numpy as np
    from oracle import darknet_oracle as orc
    import models
    from b200yolo import cfggen
    from utils.parse_config import parse_model_cfg_text
    avail = host_threads()
    defs = parse_model_cfg_text(cfggen.cfg_text(name))[1:]
    import contextlib
    with contextlib.redirect_stdout(sys.stderr):
        sd = orc.synth_state_dict(models.Darknet(cfg_for(name, 99)).state_dict(), 0)
    if threads is None:
        # "all the host threads it can use": more threads than physically free cores make torch's CPU convs slower,
        # so take the fastest of a few thread counts on a small probe forward
        best = None
        probe = orc.synth_images(1, 256, 256, seed=1)
        for t in sorted({avail, min(avail, 64), min(avail, 32), min(avail, 16), min(avail, 8)}, reverse=True):
            torch.set_num_threads(t)
            with torch.no_grad():
                orc.darknet_forward(defs, sd, probe, name)
                t0 = time.time()
                orc.darknet_forward(defs, sd, probe, name)
                dt = time.time() - t0
            if best is None or dt < best[0]:
                best = (dt, t)
        threads = best[1]
    torch.set_num_threads(threads)
    x = orc.synth_images(batch, SIZE, SIZE, seed=0)
    if kind == "train":
        for k, v in sd.items():
            if v.dtype.is_floating_point and not k.endswith(('running_mean', 'running_var')):
                v.requires_grad_(True)
        ys = [d for d in defs if d['type'] == 'yolo']
        strides = orc.yolo_strides(name, len(ys))
        av = [torch.as_tensor(np.asarray(d['anchors'])[d['mask']], dtype=torch.float32) / s
              for d, s in zip(ys, strides)]
        tg = orc.synth_targets(batch, 8, 80, seed=1)
        hyp = dict(orc.DEFAULT_HYP)

        def one():
            for v in sd.values():
                if v.requires_grad:
                    v.grad = None
            p, _ = orc.darknet_forward(defs, sd, x, name, training=True)
            loss, _ = orc.compute_loss(p, tg, av, hyp, 80, 1.0)
            loss.backward()
        what = "%s training step (forward + compute_loss + backward)" % name
    else:
        def one():
            with torch.no_grad():
                orc.darknet_forward(defs, sd, x, name)
        what = "%s eval forward" % name
    t0 = time.time()
    one()                                                     # warm-up (also sizes the sample)
    warm = time.time() - t0
    iters = max(1, min(max_iters, int(max_seconds / max(warm, 1e-3))))
    t0 = time.time()
    for _ in range(iters):
        one()
    dt = (time.time() - t0) / iters
    return {"value": batch / dt, "unit": "images/s", "cores": threads, "kind": "port",
            "sample": "%d x %s, batch %d, 640x640, fp32 torch CPU (oracle/darknet_oracle.py), after 1 warm-up"
                      % (iters, what, batch), "ms_per_step": dt * 1e3}


def torch_gpu_baseline(dev, batch, iters=5):
    """INFORMATIONAL (BASELINE.md section 3: "the kernel to beat"): the reference's own op sequence -- the oracle port --
    executed by stock PyTorch on the same GPU (eager ATen + cuDNN, autocast fp16, channels_last), yolov4 forward +
    compute_loss + backward of `batch` images at 640x640 (no optimiser step, no all-reduce).  Part of the baseline leg:
    never on the product path, never used to compute `value`."""
    sys.path.insert(0, ROOT)
    import contextlib
    import numpy as np
    from oracle import darknet_oracle as orc
    import models
    from b200yolo import cfggen
    from utils.parse_config import parse_model_cfg_text
    name = TRAIN_MODEL
    defs = parse_model_cfg_text(cfggen.cfg_text(name))[1:]
    with contextlib.redirect_stdout(sys.stderr):
        sd = orc.synth_state_dict(models.Darknet(cfg_for(name, 98)).state_dict(), 0)
    for k in list(sd):
        v = sd[k].to(dev)
        if v.dim() == 4:
            v = v.contiguous(memory_format=torch.channels_last)
        if v.dtype.is_floating_point and not k.endswith(('running_mean', 'running_var')):
            v.requires_grad_(True)
        sd[k] = v
    ys = [d for d in defs if d['type'] == 'yolo']
    strides = orc.yolo_strides(name, len(ys))
    av = [(torch.as_tensor(np.asarray(d['anchors'])[d['mask']], dtype=torch.float32) / s).to(dev) for d, s in zip(ys, strides)]
    x = orc.synth_images(batch, SIZE, SIZE, seed=0).to(dev).contiguous(memory_format=torch.channels_last)
    tg = orc.synth_targets(batch, 8, 80, seed=1).to(dev)
    hyp = dict(orc.DEFAULT_HYP)

    def one():
        for v in sd.values():
            if v.requires_grad:
                v.grad = None
        with torch.autocast("cuda", dtype=torch.float16):
            p, _ = orc.darknet_forward(defs, sd, x, name, training=True)
        loss, _ = orc.compute_loss([pi.float() for pi in p], tg, av, hyp, 80, 1.0)
        loss.backward()

    for _ in range(2):
        one()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        one()
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / iters
    return {"value": batch / (ms / 1e3), "unit": "images/s", "ms_per_step": ms,
            "what": "oracle port (the reference's op sequence) on stock PyTorch %s eager + cuDNN on this %s, autocast "
                    "fp16, channels_last: yolov4 forward + compute_loss + backward, %d images 640x640, no optimiser step"
                    % (torch.__version__, torch.cuda.get_device_name(dev), batch)}


def run_reference_arm(args, rank, world):
    if rank != 0:
        return
    # a "step" of the reference arm = one yolov4 640x640 training step of a 2-image batch on all host cores; the
    # number of timed steps is capped so that the whole run stays within a few minutes (stated in cpu_baseline.sample)
    base = cpu_reference_rate("train", TRAIN_MODEL, max_seconds=120.0, batch=2, max_iters=max(1, args.steps))
    line = {"impl": "reference", "metric": "images/sec (640x640) yolov4 training", "value": base["value"],
            "unit": "images/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": base["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": "yolov4.cfg training step 640x640 (BASELINE configs[2] per-GPU slice: 8 images / "
                                   "GPU); CPU sample batch 2", "global_batch": 2},
            "cpu_baseline": {k: base[k] for k in ("value", "unit", "cores", "kind", "sample")},
            "e2e": {"value": base["value"], "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line), flush=True)


# ----------------------------------------------------------------------------------------------------------------
# measurement helpers
# ----------------------------------------------------------------------------------------------------------------
class Dist:
    def __init__(self, world, dev):
        self.world, self.dev = world, dev

    def barrier(self):
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    def max_ms(self, ms):
        t = torch.tensor([ms], device=self.dev, dtype=torch.float64)
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())


def timed(fn, steps, dd):
    """K calls of fn bracketed by barrier + synchronize on both sides, CUDA events, max over ranks -> ms per call."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dd.barrier()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    dd.barrier()
    return dd.max_ms(e0.elapsed_time(e1)) / steps


def conv_desc_flops(name, args):
    d = args[0]._obj                      # ctypes byref(ConvDesc)
    return 2.0 * d.batch * d.out_h * d.out_w * d.out_c * d.in_c * d.ksize * d.ksize


def record_calls(fn):
    """Run fn once with the C-ABI launch recorder on; returns the list of (name, args)."""
    from b200yolo import lib
    lib.RECORD = []
    try:
        fn()
        torch.cuda.synchronize()
        return lib.RECORD
    finally:
        lib.RECORD = None


def replay_convs(calls, iters):
    """Replay the wgmma convolution launches of one recorded step back to back -> (ms per step-worth, FLOPs, n)."""
    from b200yolo import lib
    convs = [(n, a) for (n, a) in calls if n in CONV_CALLS]
    flops = sum(conv_desc_flops(n, a) for n, a in convs)
    raw = lib.raw()
    cur = lib.stream_ptr()          # launches may have been recorded on a side stream: replay all on the timed stream
    fns = [(getattr(raw, n), a[:-1] + (cur,)) for n, a in convs]
    for f, a in fns:
        f(*a)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        for f, a in fns:
            f(*a)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters, flops, len(convs)


def roofline_block(conv_ms, conv_flops, n_convs, step_ms, what):
    pk = peaks()
    achieved = conv_flops / (conv_ms / 1e3) / 1e12
    return {"bound": "tensor", "achieved": achieved, "peak": pk["tflops"], "unit": "TFLOP/s",
            "frac": achieved / pk["tflops"], "peak_source": pk["source"],
            "kernel": "wgmma conv family (%s): %d launches of one step replayed back to back" % (what, n_convs),
            "kernel_ms_per_step": conv_ms, "share_of_step": conv_ms / step_ms,
            "algorithmic_flops_per_step": conv_flops,
            "whole_step_frac": conv_flops / (step_ms / 1e3) / 1e12 / pk["tflops"]}


# ----------------------------------------------------------------------------------------------------------------
# primary workload: YOLOv4 training step, data parallel
# ----------------------------------------------------------------------------------------------------------------
def note(rank, msg):
    """progress marker on stderr (per rank): the log shows how far a failing multi-GPU run got"""
    sys.stderr.write("[bench.py rank %d] %s\n" % (rank, msg))
    sys.stderr.flush()


DUMP_SAMPLE = 1 << 20          # elements kept per large output (fixed, seeded positions)


def dump_outputs(d, items, pred, flat_grad):
    """The last timed step's results as .npy files: the four loss items, and for each prediction tensor and the flat
    fp32 gradient buffer a fixed seeded sample of DUMP_SAMPLE elements (float32, with their positions as float64) plus
    the float64 sum of the whole tensor (about 50 MB in all)."""
    import numpy as np
    os.makedirs(d, exist_ok=True)
    torch.cuda.synchronize()
    arrays = {"loss_items": items.detach().float().cpu()}
    for name, t in [("pred%d" % i, p) for i, p in enumerate(pred)] + [("flat_grad", flat_grad)]:
        flat = t.detach().float().reshape(-1)
        if flat.numel() > DUMP_SAMPLE:
            g = torch.Generator().manual_seed(1234 + flat.numel())
            idx = torch.randperm(flat.numel(), generator=g)[:DUMP_SAMPLE].sort().values
            arrays[name + "_sample"] = flat[idx.to(flat.device)].cpu()
            arrays[name + "_sample_index"] = idx.double()
        else:
            arrays[name] = flat.cpu()
        arrays[name + "_sum"] = flat.double().sum().reshape(1).cpu()
    for name, a in arrays.items():
        np.save(os.path.join(d, name + ".npy"), a.numpy())


def run_train(args, dev, rank, world, dd):
    import torch.distributed as dist
    from b200yolo.parallel import FlatDataParallel
    from utils import utils as my_utils
    B = args.train_batch
    model = build_model(TRAIN_MODEL, dev, rank, train=True)
    note(rank, "model built")
    dp = FlatDataParallel(model)
    note(rank, "flat data-parallel buffers ready (world %d)" % world)
    u8, tg = synth_batch(B, 100 + rank)
    host_u8, host_t = u8.pin_memory(), tg.pin_memory()
    x_dev = (host_u8.to(dev).float() / 256.0).contiguous()
    t_dev = host_t.to(dev)
    lr, scale = 1e-4, B * world / 64.0                    # train.py:437  loss *= batch_size / 64 (global batch)
    state = {"items": None}

    def step(x, t):
        dp.zero_grad()
        pred, _ = dp(x)
        loss, items = my_utils.compute_loss(pred, t, dp)
        (loss * scale).backward()
        dp.reduce_gradients()
        dp.step(lr=lr, momentum=0.937, weight_decay=0.000484)
        state["items"] = items
        state["pred"] = pred

    for _ in range(args.warmup):
        step(x_dev, t_dev)
    torch.cuda.synchronize()
    note(rank, "warm-up done")

    sampler = ClockSampler(dev.index)
    sampler.start()
    ms_step = timed(lambda: step(x_dev, t_dev), args.steps, dd)
    clocks = sampler.stop()
    value = world * B / (ms_step / 1e3)
    items = [float(v) for v in state["items"]]
    note(rank, "timed region done: %.3f ms/step" % ms_step)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, state["items"], state["pred"], dp.flat_grad)

    # ---- end to end: pinned host uint8 batch + targets -> H2D -> /256 -> step -> D2H of the loss items ----------
    copy_stream = torch.cuda.Stream()
    dev_u8 = [torch.empty_like(host_u8, device=dev) for _ in range(2)]
    dev_t = [torch.empty_like(host_t, device=dev) for _ in range(2)]
    ready = [torch.cuda.Event() for _ in range(2)]
    consumed = [torch.cuda.Event() for _ in range(2)]
    main = torch.cuda.current_stream()
    items_host = torch.empty(4, dtype=torch.float32).pin_memory()

    def issue_copy(j):
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[j])
            dev_u8[j].copy_(host_u8, non_blocking=True)
            dev_t[j].copy_(host_t, non_blocking=True)
            ready[j].record(copy_stream)

    for j in range(2):
        consumed[j].record(main)
    issue_copy(0)
    cnt = {"i": 0}

    def e2e_step():
        j = cnt["i"] & 1
        main.wait_event(ready[j])
        x = dev_u8[j].float() / 256.0                      # train.py:348
        step(x, dev_t[j])
        consumed[j].record(main)
        issue_copy(j ^ 1)                                  # prefetch the next batch while this one computes
        items_host.copy_(state["items"], non_blocking=True)
        cnt["i"] += 1

    for _ in range(3):
        e2e_step()
    ms_e2e = timed(e2e_step, args.steps, dd)
    e2e_value = world * B / (ms_e2e / 1e3)

    # ---- the exchange step alone (N > 1): one all-reduce of the flat fp32 gradient buffer -------------------------
    allreduce = None
    if world > 1:
        ms_ar = timed(lambda: dp.reduce_gradients(), 5, dd)
        nbytes = dp.flat_grad.numel() * 4
        allreduce = {"ms": ms_ar, "bytes": nbytes, "algbw_gbs": nbytes / ms_ar / 1e6,
                     "busbw_gbs": nbytes / ms_ar / 1e6 * 2 * (world - 1) / world}

    # ---- roofline of the dominant kernel family: record one eager step, replay its conv launches ----------------
    saved = getattr(model, "use_cuda_graph", None)
    model.use_cuda_graph = False
    try:
        calls = record_calls(lambda: step(x_dev, t_dev))
    finally:
        if saved is None:
            del model.use_cuda_graph
        else:
            model.use_cuda_graph = saved
    conv_ms, conv_flops, n_convs = replay_convs(calls, iters=args.steps)
    roofline = roofline_block(conv_ms, conv_flops, n_convs, ms_step, "forward + data gradient + weight gradient")
    roofline["table_flops_per_step"] = FLOPS_TRAIN[TRAIN_MODEL] * B
    launches = len(calls)
    return {"value": value, "ms_per_step": ms_step, "clocks": clocks, "roofline": roofline, "allreduce": allreduce,
            "e2e": {"value": e2e_value, "unit": "images/s", "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": int(host_u8.numel() + host_t.numel() * 4), "d2h_bytes_per_step": 16,
                    "result": "the four loss items (lbox, lobj, lcls, loss) of the step, what train.py logs"},
            "gpu_launches": launches * args.steps, "launches_per_step": launches, "loss_items": items,
            "grad_bytes": int(dp.flat_grad.numel() * 4), "batch": B}


# ----------------------------------------------------------------------------------------------------------------
# secondary workloads: inference replicas (configs[1] and YOLOv4)
# ----------------------------------------------------------------------------------------------------------------
def run_infer(name, args, dev, rank, world, dd, with_e2e=True):
    B = INFER_BATCH
    model = build_model(name, dev, rank, train=False)
    u8, _ = synth_batch(B, 200 + rank)
    host_u8 = u8.pin_memory()
    x_dev = (host_u8.to(dev).float() / 256.0).contiguous()
    out = {}
    with torch.no_grad():
        for _ in range(max(3, args.warmup)):
            io, p, _ = model(x_dev)
        torch.cuda.synchronize()
        ms_step = timed(lambda: model(x_dev), args.steps, dd)
        out["value"] = world * B / (ms_step / 1e3)
        out["ms_per_step"] = ms_step
        if with_e2e:
            no = io.shape[-1]
            top_host = torch.empty((B, no), dtype=torch.float32).pin_memory()
            copy_stream = torch.cuda.Stream()
            dev_u8 = [torch.empty_like(host_u8, device=dev) for _ in range(2)]
            ready = [torch.cuda.Event() for _ in range(2)]
            consumed = [torch.cuda.Event() for _ in range(2)]
            main = torch.cuda.current_stream()

            def issue_copy(j):
                with torch.cuda.stream(copy_stream):
                    copy_stream.wait_event(consumed[j])
                    dev_u8[j].copy_(host_u8, non_blocking=True)
                    ready[j].record(copy_stream)

            for j in range(2):
                consumed[j].record(main)
            issue_copy(0)
            cnt = {"i": 0}

            def e2e_step():
                j = cnt["i"] & 1
                main.wait_event(ready[j])
                # uint8 batch straight into the model: the stem kernel applies the reference's "/ 256.0"
                o, _, _ = model(dev_u8[j])
                consumed[j].record(main)
                issue_copy(j ^ 1)
                idx = o[..., 4].argmax(dim=1)                              # best-objectness row per image
                top_host.copy_(o[torch.arange(B, device=dev), idx], non_blocking=True)
                cnt["i"] += 1

            for _ in range(3):
                e2e_step()
            ms2 = timed(e2e_step, args.steps, dd)
            out["e2e"] = {"value": world * B / (ms2 / 1e3), "unit": "images/s",
                          "h2d_bytes_per_step": int(host_u8.numel()), "d2h_bytes_per_step": int(top_host.numel() * 4),
                          "result": "the top-objectness decoded row per image (a stand-in for post-NMS detections)"}
        saved = getattr(model, "use_cuda_graph", None)
        model.use_cuda_graph = False
        try:
            calls = record_calls(lambda: model(x_dev))
        finally:
            if saved is None:
                del model.use_cuda_graph
            else:
                model.use_cuda_graph = saved
        conv_ms, conv_flops, n_convs = replay_convs(calls, iters=args.steps)
        out["roofline"] = roofline_block(conv_ms, conv_flops, n_convs, ms_step, "forward")
        out["launches_per_step"] = len(calls)
        out["workload"] = "%s.cfg inference bs=%d 640x640 per GPU, fp16 fused conv path" % (name, B)
    del model
    torch.cuda.empty_cache()
    return out


def run_nms(args, dev, dd):
    """Secondary block (SURVEY 8 f1): non_max_suppression + TP matching of a batch of 32 x 25 200 x 85 predictions with
    the statistics of a trained detector at test.py's conf_thres 0.001 (synthetic: ~60 objects per image, each a cluster
    of jittered boxes, a few per cent of background rows above the threshold; random-weight predictions would make
    every one of the 2 M (row, class) pairs a candidate, which the reference cannot process either)."""
    from b200yolo import detect
    B, R, nc = INFER_BATCH, 25200, 80
    g = torch.Generator(device=dev).manual_seed(11)
    p = torch.zeros((B, R, 5 + nc), device=dev)
    p[..., 0:2] = torch.rand((B, R, 2), device=dev, generator=g) * SIZE
    p[..., 2:4] = torch.exp(torch.rand((B, R, 2), device=dev, generator=g) * 4.0 + 1.0)
    p[..., 4] = torch.rand((B, R), device=dev, generator=g) * 0.0009               # background: below conf_thres
    p[..., 5:] = torch.rand((B, R, nc), device=dev, generator=g) * 0.001           # obj * cls stays below it
    n_obj, per = 60, 40
    rows = torch.stack([torch.randperm(R, device=dev, generator=g)[:n_obj * per] for _ in range(B)])
    ctr = (torch.rand((B, n_obj, 1, 2), device=dev, generator=g) * (SIZE - 140) + 70)
    wh = torch.exp(torch.rand((B, n_obj, 1, 2), device=dev, generator=g) * 2.5 + 2.5)
    box = torch.cat((ctr + torch.randn((B, n_obj, per, 2), device=dev, generator=g) * 0.06 * wh,
                     wh * torch.exp(torch.randn((B, n_obj, per, 2), device=dev, generator=g) * 0.08)), 3)
    obj = torch.rand((B, n_obj, per), device=dev, generator=g) * 0.9 + 0.05
    cls = torch.randint(0, nc, (B, n_obj, 1), device=dev, generator=g).expand(B, n_obj, per)
    bi = torch.arange(B, device=dev)[:, None].expand(B, n_obj * per)
    p[bi, rows, 0:4] = box.reshape(B, -1, 4)
    p[bi, rows, 4] = obj.reshape(B, -1)
    p[bi, rows, 5 + cls.reshape(B, -1)] = torch.rand((B, n_obj * per), device=dev, generator=g) * 0.7 + 0.3
    extra = torch.rand((B, R), device=dev, generator=g) < 0.02                     # weak background detections
    extra &= p[..., 4] < 0.001
    p[..., 4] = torch.where(extra, torch.rand((B, R), device=dev, generator=g) * 0.05, p[..., 4])
    ecls = torch.randint(0, nc, (B, R), device=dev, generator=g)
    p[..., 5:].scatter_(2, ecls[..., None], torch.where(extra, 0.9, 0.0005)[..., None].to(p.dtype))
    targets = torch.cat([torch.cat((torch.full((n_obj, 1), float(b), device=dev), cls[b, :, :1].float(),
                                    (ctr[b, :, 0] / SIZE), (wh[b, :, 0] / SIZE)), 1) for b in range(B)])
    iouv = torch.linspace(0.5, 0.95, 10)

    def step():
        packed = detect.nms_packed(p, conf_thres=0.001, iou_thres=0.6)
        detect.match_batch(packed, targets, SIZE, SIZE, iouv)
        return packed

    for _ in range(3):
        packed = step()
    ms = timed(step, args.steps, dd)
    return {"value": B / (ms / 1e3), "unit": "images/s", "ms_per_step": ms,
            "candidates_per_image": sum(torch.diff(packed.offsets_dev).tolist()) / B,
            "detections_per_image": sum(packed.counts) / B, "launches_per_step": 10,
            "workload": "non_max_suppression (conf 0.001, iou 0.6, multi-label, merge) + TP matching, batch %d x %d rows x "
                        "%d classes resident in HBM, synthetic trained-detector statistics; includes the two host reads "
                        "of the candidate / detection counts" % (B, R, nc)}


def run_tool_block(script, extra, what, timeout=120, env=None):
    """Secondary block measured by one of the repo's stand-alone benchmark tools in its OWN process (tools/*.py print one
    JSON line): a failure or a hang there cannot touch the headline that was measured above."""
    cmd = [sys.executable, os.path.join(ROOT, "tools", script)] + list(extra)
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout,
                           env=dict(os.environ, **env) if env else None)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
        if r.returncode != 0 or not lines:
            tail = (r.stderr or r.stdout).strip().splitlines()[-1:] or [""]
            return {"error": "%s exited with %d: %s" % (script, r.returncode, tail[0][:300])}
        d = json.loads(lines[-1])
    except subprocess.TimeoutExpired:
        return {"error": "%s: no result within %d s" % (script, timeout)}
    except Exception as e:          # a secondary block must never take the headline down
        return {"error": "%s: %s: %s" % (script, type(e).__name__, str(e)[:300])}
    out = {k: d[k] for k in ("value", "unit", "ms_per_step") if k in d}
    out["workload"] = what
    out["measured_by"] = "tools/%s %s (own process%s)" % (script, " ".join(extra),
                                                          ", " + " ".join("%s=%s" % kv for kv in env.items()) if env else "")
    for k in ("loss_items", "calibration", "dtype"):
        if k in d:
            out[k] = d[k]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--train-batch", type=int, default=TRAIN_BATCH, help="images per GPU of the training workload")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed training step's outputs as DIR/<name>.npy")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))

    if args.impl == "reference":
        run_reference_arm(args, rank, world)
        return
    if args.gpus > 1 and world == 1 and "RANK" not in os.environ:
        # plain `python bench.py --gpus N`: start one process per GPU ourselves
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus),
               "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 2000)] + sys.argv
        rc = subprocess.call(cmd)
        if rc != 0:
            sys.stderr.write("[bench.py] torchrun exited with status %d\n" % rc)
        raise SystemExit(rc)

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (H100): the hot path has no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    import torch.distributed as dist
    if world > 1:
        dist.init_process_group("nccl", init_method="env://", device_id=dev)
    dd = Dist(world, dev)

    tr = run_train(args, dev, rank, world, dd)

    secondary = {}
    if world == 1 and not args.no_secondary:
        # free the training plan before the inference replicas are built
        torch.cuda.empty_cache()
        for name in ("yolov3", "yolov4"):
            try:
                secondary["%s_infer_bs%d" % (name, INFER_BATCH)] = run_infer(name, args, dev, rank, world, dd)
            except Exception as e:  # a secondary block must not take the headline down
                secondary["%s_infer_bs%d" % (name, INFER_BATCH)] = {"error": "%s: %s" % (type(e).__name__, e)}
        try:
            secondary["nms_bs%d" % INFER_BATCH] = run_nms(args, dev, dd)
        except Exception as e:
            secondary["nms_bs%d" % INFER_BATCH] = {"error": "%s: %s" % (type(e).__name__, str(e)[:300])}
        # the two remaining BASELINE configurations, per-GPU slices, each in its own process
        torch.cuda.empty_cache()
        mb_args = ["--model", "yolov3-mobilenet", "--batch", "32", "--size", str(SIZE), "--steps", str(args.steps)]
        mb_what = ("yolov3-mobilenet.cfg (depthwise-separable backbone) training step, 32 images / GPU, 640x640: forward + "
                   "YOLO loss + backward + gradient exchange + fused SGD-Nesterov (BASELINE configs[3]: bs 128 on 4 GPUs)")
        blk = run_tool_block("bench_train.py", mb_args, mb_what)
        if "error" in blk:          # second attempt with eager launches instead of CUDA-graph replay
            first = blk["error"]
            blk = run_tool_block("bench_train.py", mb_args, mb_what, env={"B2Y_NO_GRAPH": "1"})
            blk["first_attempt"] = first
        secondary["yolov3_mobilenet_train_bs32"] = blk
        secondary["yolov3_int8_ptq_infer_bs%d" % INFER_BATCH] = run_tool_block(
            "bench_ptq_native.py", ["--batch", str(INFER_BATCH), "--size", str(SIZE), "--steps", str(args.steps)],
            "yolov3.cfg INT8 PTQ inference bs=%d 640x640 (BASELINE configs[4] at the batch of configs[1]): native "
            "calibration, then the int8 wgmma graph" % INFER_BATCH)

    cpu, tgpu = None, None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cpu = cpu_reference_rate("train", TRAIN_MODEL, max_seconds=20.0, batch=2, max_iters=3)
        cpu = {k: cpu[k] for k in ("value", "unit", "cores", "kind", "sample")}
        try:
            torch.cuda.empty_cache()
            tgpu = torch_gpu_baseline(dev, tr["batch"], iters=args.steps)
        except Exception as e:      # informational only
            tgpu = {"error": "%s: %s" % (type(e).__name__, str(e)[:200])}

    if rank == 0:
        B = tr["batch"]
        line = {
            "metric": "images/sec (640x640) yolov4 training", "value": tr["value"], "unit": "images/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": tr["ms_per_step"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f16", "data": "synthetic",
            "config": {"workload": "yolov4.cfg (CSPDarknet-53 + Mish) training step, %d images / GPU, 640x640: "
                                   "forward + YOLO loss + backward + ONE NCCL all-reduce of the flat fp32 gradients + "
                                   "fused SGD-Nesterov (BASELINE configs[2]: bs 64 on 8 GPUs)" % B,
                       "global_batch": B * world, "parallelism": "dp%d" % world,
                       "precision": "fp16 activations / weights, bf16 activation gradients, fp32 accumulation, "
                                    "statistics, weight gradients, master weights and optimiser",
                       "l2": "activations + gradients of one step (> 8 GB) exceed the 50 MB L2; every step re-reads "
                             "them from HBM",
                       "cuda_graph": True, "grad_allreduce_bytes": tr["grad_bytes"],
                       "launches_per_step": tr["launches_per_step"], "loss_items": tr["loss_items"]},
            "gpu": torch.cuda.get_device_name(dev),
            "clocks": tr["clocks"],
            "e2e": tr["e2e"],
            "gpu_launches": tr["gpu_launches"],
            "roofline": tr["roofline"],
        }
        if tr["allreduce"] is not None:
            line["allreduce"] = tr["allreduce"]
        if cpu is not None:
            line["cpu_baseline"] = cpu
        if tgpu is not None:
            line["torch_gpu_baseline"] = tgpu
        if secondary:
            line["secondary"] = secondary
        print(json.dumps(line), flush=True)
    note(rank, "done")
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    try:
        main()
    except SystemExit:
        raise
    except BaseException:
        # torchrun swallows per-rank tracebacks (error_file: <N/A>): print them with the rank
        sys.stderr.write("[bench.py rank %s]\n%s\n" % (os.environ.get("RANK", "0"), traceback.format_exc()))
        raise
