"""Time the device evaluation loader (b200yolo.preprocess.DeviceEvalLoader) against a CPU arm that makes the cv2 calls
of LoadImagesAndLabels(rect=True) + collate_fn in worker processes, on the same synthetic JPEG files.

    python tools/time_eval_loader.py [--sizes 416 640] [--batch 32] [--batches 4] [--workers 8] [--out DIR]

Device arm, per batch: `decode` = cv2.imread of the batch on host threads plus the host plan (sizes, border, labels);
`device` = one host-to-device copy of the raw sources and item table, the b2y_load_batch_u8 launch and the targets copy,
ended by a device synchronise.  CPU arm, per batch: imread, INTER_AREA resize (sources larger than img_size),
copyMakeBorder to the batch shape, channel flip + transpose in N worker processes, then np.stack in the parent, as
test.py's DataLoader workers and collate_fn do.  Prints one JSON line with the card, its power limit and the host CPU.
"""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200")
sys.path.insert(0, PKG)

COCO_LIKE = [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (500, 375), (640, 640), (360, 640), (612, 612),
             (424, 640), (640, 512), (333, 500)]


def write_dataset(d, n, seed):
    import cv2
    rng = np.random.default_rng(seed)
    files = []
    for i in range(n):
        h, w = COCO_LIKE[int(rng.integers(len(COCO_LIKE)))]
        y, x = np.mgrid[0:h, 0:w]
        base = np.stack([(x * (1 + c) + y * (3 - c)) % 256 for c in range(3)], -1)
        img = np.clip(base + rng.integers(-20, 21, (h, w, 3)), 0, 255).astype(np.uint8)
        f = os.path.join(d, "im%04d.jpg" % i)
        cv2.imwrite(f, img, [cv2.IMWRITE_JPEG_QUALITY, 90])
        files.append((f, h, w))
    return files


class Dataset:
    """The attributes of LoadImagesAndLabels(rect=True, augment=False): files sorted by aspect ratio, rect batch shapes."""

    def __init__(self, files, img_size, bs):
        ar = np.array([h / w for _, h, w in files])
        order = ar.argsort()
        self.img_files = [files[i][0] for i in order]
        ar = ar[order]
        n = len(files)
        self.batch = np.floor(np.arange(n) / bs).astype(int)
        shapes = []
        for b in range(self.batch[-1] + 1):
            a = ar[self.batch == b]
            shapes.append([a.max(), 1] if a.max() < 1 else ([1, 1 / a.min()] if a.min() > 1 else [1, 1]))
        self.batch_shapes = np.ceil(np.array(shapes) * img_size / 32.).astype(int) * 32
        rng = np.random.default_rng(1)
        self.labels = [np.concatenate([rng.integers(0, 80, (k, 1)), rng.uniform(0.2, 0.8, (k, 2)),
                                       rng.uniform(0.05, 0.3, (k, 2))], 1).astype(np.float32)
                       for k in rng.integers(0, 8, n)]
        self.img_size, self.imgs, self.is_gray_scale, self.augment, self.rect = img_size, [None] * n, False, False, True


def cpu_load(args):
    import cv2
    path, img_size, shape = args
    img = cv2.imread(path)
    h0, w0 = img.shape[:2]
    r = img_size / max(h0, w0)
    if r < 1:
        img = cv2.resize(img, (int(w0 * r), int(h0 * r)), interpolation=cv2.INTER_AREA)
    h, w = img.shape[:2]
    dh, dw = (shape[0] - h) / 2, (shape[1] - w) / 2
    top, bottom, left, right = int(round(dh - 0.1)), int(round(dh + 0.1)), int(round(dw - 0.1)), int(round(dw + 0.1))
    img = cv2.copyMakeBorder(img, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
    return np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1))


def device_info():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit_and_max_sm_clock"] = q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = None
    cpu = None
    try:
        with open("/proc/cpuinfo") as f:
            cpu = next((ln.split(":", 1)[1].strip() for ln in f if ln.startswith("model name")), None)
    except OSError:
        pass
    info["host_cpu"] = cpu
    info["host_cpus"] = os.cpu_count()
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[416, 640])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_eval_loader.py measures on a CUDA device; none found")
    from b200yolo.preprocess import DeviceEvalLoader
    result = dict(device_info(), batch=a.batch, batches=a.batches, workers=a.workers, arms={})
    with tempfile.TemporaryDirectory(prefix="b2y_evalload_") as d:
        files = write_dataset(d, a.batch * a.batches, seed=0)
        pool = mp.get_context("spawn").Pool(a.workers)
        try:
            for size in a.sizes:
                ds = Dataset(files, size, a.batch)
                loader = DeviceEvalLoader(ds, a.batch)
                jobs = [[(ds.img_files[i], size, tuple(int(v) for v in ds.batch_shapes[ds.batch[i]]))
                         for i in range(b * a.batch, (b + 1) * a.batch)] for b in range(len(loader))]
                # warm-up: every batch shape once in each arm (module load, allocator, worker start)
                for b in range(len(loader)):
                    loader.batch(b)
                    np.stack(pool.map(cpu_load, jobs[b]), 0)
                torch.cuda.synchronize()
                dec, dev, cpu = [], [], []
                for _ in range(a.repeats):
                    for b in range(len(loader)):
                        t0 = time.perf_counter()
                        plans = loader.host_batch(b)
                        t1 = time.perf_counter()
                        loader.device_batch(plans)
                        torch.cuda.synchronize()
                        t2 = time.perf_counter()
                        np.stack(pool.map(cpu_load, jobs[b]), 0)
                        t3 = time.perf_counter()
                        dec.append(t1 - t0)
                        dev.append(t2 - t1)
                        cpu.append(t3 - t2)
                med = lambda v: round(1e3 * float(np.median(v)), 3)  # noqa: E731
                result["arms"][str(size)] = dict(device_decode_ms=med(dec), device_stage_ms=med(dev),
                                                 device_total_ms=med(np.add(dec, dev)), cpu_workers_ms=med(cpu),
                                                 batch_shapes=[[int(v) for v in s] for s in ds.batch_shapes])
        finally:
            pool.close()
            pool.join()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_eval_loader.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
