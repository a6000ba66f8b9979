"""Time the device training loader (b200yolo.preprocess.DeviceTrainLoader) against a CPU arm that makes the cv2 calls
of LoadImagesAndLabels(augment=True).__getitem__ + collate_fn in worker processes, on the same synthetic JPEG files.

    python tools/time_train_loader.py [--size 640] [--batches-of 8 32] [--steps 4] [--out DIR]

Both arms run with an image cache (train.py's cache_images=True: load_image's INTER_LINEAR tiles kept in host memory)
and without one (cv2.imread + INTER_LINEAR per tile).  Device arm, per batch: `plan` = the random draws, decoding of
the batch's distinct images on host threads (uncached) and the host plan (rectangles, affine map, LUTs, labels);
`device` = one host-to-device copy of the sources and both item tables, b2y_mosaic_u8 and b2y_affine_hsv_u8 and the
targets copy, ended by a device synchronise.  CPU arm, per batch: for each item, the 4 tiles, the 2s x 2s canvas,
cv2.warpAffine, the two cv2.cvtColor and three LUTs, the flip and the channel shuffle in min(cpus, batch, 8) forked
worker processes (the draws are the device arm's, so both arms do the same work), then np.stack in the parent.  Prints
one JSON line with the card, its power limit and the host CPU.
"""
import argparse
import json
import multiprocessing as mp
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200")
sys.path.insert(0, PKG)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_eval_loader import device_info, write_dataset  # noqa: E402

HYP = dict(hsv_h=0.0138, hsv_s=0.678, hsv_v=0.36, degrees=0.0, translate=0.0, scale=0.0, shear=0.0)  # train.py's
_DS = None                                                       # the dataset the forked workers read


class Dataset:
    """The attributes of LoadImagesAndLabels(augment=True, rect=False) the loaders read."""

    def __init__(self, files, img_size, cache):
        import cv2
        from b200yolo.preprocess import train_tile_size
        n = len(files)
        self.img_files = [f for f, _, _ in files]
        self.n, self.img_size, self.hyp, self.is_gray_scale = n, img_size, HYP, False
        self.augment, self.rect, self.image_weights = True, False, False
        rng = np.random.default_rng(1)
        self.labels = [np.concatenate([rng.integers(0, 80, (k, 1)), rng.uniform(0.2, 0.8, (k, 2)),
                                       rng.uniform(0.05, 0.3, (k, 2))], 1).astype(np.float32)
                       for k in rng.integers(0, 8, n)]
        self.imgs = [None] * n
        if cache:
            self.img_hw0, self.img_hw = [], []
            for i, f in enumerate(self.img_files):
                img = cv2.imread(f)
                h0, w0 = img.shape[:2]
                h, w = train_tile_size(h0, w0, img_size)
                self.imgs[i] = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR) if (h, w) != (h0, w0) else img
                self.img_hw0.append((h0, w0))
                self.img_hw.append((h, w))

    def __len__(self):
        return self.n


def cpu_item(job):
    """One item as __getitem__ builds it, from the draws of the device arm's plan."""
    import cv2
    from b200yolo.preprocess import train_tile_size
    tiles, rects, M, lut, flip = job
    ds, s = _DS, _DS.img_size
    img4 = np.full((2 * s, 2 * s, 3), 114, dtype=np.uint8)
    for i, ((x1a, y1a, x2a, y2a), (dx, dy)) in zip(tiles, rects):
        img = ds.imgs[i]
        if img is None:
            img = cv2.imread(ds.img_files[i])
            h, w = train_tile_size(img.shape[0], img.shape[1], s)
            if (h, w) != img.shape[:2]:
                img = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
        img4[y1a:y2a, x1a:x2a] = img[y1a + dy:y2a + dy, x1a + dx:x2a + dx]
    img = cv2.warpAffine(img4, M[:2], dsize=(s, s), flags=cv2.INTER_LINEAR, borderValue=(114, 114, 114))
    hue, sat, val = cv2.split(cv2.cvtColor(img, cv2.COLOR_BGR2HSV))
    hsv = cv2.merge((cv2.LUT(hue, lut[:256]), cv2.LUT(sat, lut[256:512]), cv2.LUT(val, lut[512:])))
    cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR, dst=img)
    if flip:
        img = np.fliplr(img)
    return np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1))


def main():
    global _DS
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--batches-of", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_train_loader.py measures on a CUDA device; none found")
    from b200yolo.preprocess import DeviceTrainLoader
    result = dict(device_info(), size=a.size, steps=a.steps, arms={})
    with tempfile.TemporaryDirectory(prefix="b2y_trainload_") as d:
        files = write_dataset(d, max(a.batches_of) * a.steps, seed=0)
        for cache in (True, False):
            _DS = Dataset(files, a.size, cache)
            for bs in a.batches_of:
                workers = min(os.cpu_count() or 1, bs, 8)
                pool = mp.get_context("fork").Pool(workers)      # the workers share the cache, as train.py's do
                try:
                    loader = DeviceTrainLoader(_DS, bs, drop_last=True)
                    batches = [idx for _, idx in zip(range(a.steps), loader._index)]
                    plans = [loader.host_batch(idx) for idx in batches]
                    for p in plans:                               # warm-up: allocator, module load, workers
                        loader.device_batch(p)
                        np.stack(pool.map(cpu_item, [(q["tiles"], q["rects"], q["M"], q["lut"], q["flip"])
                                                     for q in p[1]]), 0)
                    torch.cuda.synchronize()
                    plan_t, dev_t, cpu_t = [], [], []
                    for _ in range(a.repeats):
                        for idx in batches:
                            t0 = time.perf_counter()
                            planned = loader.host_batch(idx)
                            t1 = time.perf_counter()
                            loader.device_batch(planned)
                            torch.cuda.synchronize()
                            t2 = time.perf_counter()
                            np.stack(pool.map(cpu_item, [(q["tiles"], q["rects"], q["M"], q["lut"], q["flip"])
                                                         for q in planned[1]]), 0)
                            t3 = time.perf_counter()
                            plan_t.append(t1 - t0)
                            dev_t.append(t2 - t1)
                            cpu_t.append(t3 - t2)
                finally:
                    pool.close()
                    pool.join()
                med = lambda v: round(1e3 * float(np.median(v)), 3)  # noqa: E731
                result["arms"]["%s_b%d" % ("cache" if cache else "files", bs)] = dict(
                    device_plan_ms=med(plan_t), device_stage_ms=med(dev_t), device_total_ms=med(np.add(plan_t, dev_t)),
                    cpu_workers_ms=med(cpu_t), workers=workers)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_train_loader.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
