"""Generate tests/golden/trainloader_case.npz by RUNNING THE REFERENCE's training loader: LoadImagesAndLabels(
augment=True, rect=False) (utils/datasets.py:262-501, 511-608, 649-715: load_mosaic, random_affine, augment_hsv, the
flip) under a num_workers=0 DataLoader(shuffle=True, collate_fn) with fixed torch / random / np.random seeds, over
seeded synthetic datasets written to a temporary directory as PNG (lossless, so decoding is not a variable).  Stores,
per dataset, the source sizes and seeds (preprocess_oracle.synth_image regenerates the decoded sources), the parsed
labels, the hyp, the seeds, the image_weights indices, every batch's image bytes, targets and paths (file names), and
the three RNG states after the batches kept.  Run where the reference is (the GPU machines have none); the output is
committed.

    python oracle/gen_golden_trainloader.py
"""
import itertools
import json
import os
import random
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("B2Y_REFERENCE_ROOT", "/root/reference")
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "mpl_stub"))

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, HERE)
from preprocess_oracle import synth_image  # noqa: E402

TRAIN_HYP = dict(hsv_h=0.0138, hsv_s=0.678, hsv_v=0.36, degrees=1.98 * 0, translate=0.05 * 0, scale=0.05 * 0,
                 shear=0.641 * 0)                                   # train.py's defaults: a pure s / 2 translation
AFFINE_HYP = dict(hsv_h=0.0138, hsv_s=0.678, hsv_v=0.36, degrees=10, translate=0.1, scale=0.1, shear=10)

# name, img_size, batch_size, gray, cache, image_weights, hyp, seed, batches kept (None = the whole epoch),
# [(h0, w0, n_labels or None = no label file)].  Every dataset holds all the source kinds; only the first batches of an
# epoch are kept (the RNG states are those after them), which keeps the fixture small: the batches are noisy images
# that barely compress.
SOURCES_128 = [
    (300, 200, 3),      # larger, fractional INTER_LINEAR down -> 128 x 85
    (256, 192, 2),      # exact 2x down (cv::resize's INTER_AREA shortcut) -> 128 x 96
    (60, 90, 4),        # smaller: INTER_LINEAR up -> 85 x 128
    (128, 100, 2),      # equal: no resize
    (300, 3, 1),        # 1 pixel thin after the resize -> 128 x 1
    (200, 160, 0),      # empty label file
    (90, 140, 6),       # boxes at the edges, some dropped by the affine filter
    (170, 130, None),   # no label file
]
SOURCES_160 = [
    (320, 320, 3),      # exact 2x down
    (400, 250, 2),
    (100, 70, 5),
    (160, 160, 1),      # equal
    (2, 300, 1),        # thin
    (240, 180, 0),
    (120, 200, 6),
    (333, 222, 2),
]
DATASETS = [
    ("c128", 128, 4, False, True, False, TRAIN_HYP, 11, 1, SOURCES_128),
    ("c128u", 128, 2, False, False, False, AFFINE_HYP, 12, 2, SOURCES_128),        # RNG and canvas across batches
    ("c160", 160, 2, False, True, False, AFFINE_HYP, 13, 1, SOURCES_160),
    ("c160w", 160, 2, False, True, True, TRAIN_HYP, 14, 1, SOURCES_160),
    ("g128", 128, 4, True, False, False, AFFINE_HYP, 15, None, SOURCES_128[:6]),  # whole epoch, partial last batch
]


def synth_labels(n, seed):
    """n boxes; every third one small and against an edge, which random_affine's filter tends to drop."""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(n):
        if k % 3 == 2:
            w, h = rng.uniform(0.01, 0.05), rng.uniform(0.01, 0.05)
            x, y = (w / 2 if k % 2 else 1 - w / 2), rng.uniform(h / 2, 1 - h / 2)
        else:
            w, h = rng.uniform(0.05, 0.6), rng.uniform(0.05, 0.6)
            x, y = rng.uniform(w / 2, 1 - w / 2), rng.uniform(h / 2, 1 - h / 2)
        rows.append("%d %.6f %.6f %.6f %.6f" % (rng.integers(0, 80), x, y, w, h))
    return "\n".join(rows) + ("\n" if rows else "")


def source_seed(name, k):
    return 500 * len(name) + 31 * k + sum(map(ord, name))


def main():
    os.chdir(REF)
    np.int = int                               # datasets.py:278 still uses the alias removed from numpy
    from utils.datasets import LoadImagesAndLabels
    from utils.utils import labels_to_image_weights
    out = {}
    tmp = tempfile.mkdtemp(prefix="b2y_trainloader_")
    try:
        for name, s, bs, gray, cache, iw, hyp, seed, keep, spec in DATASETS:
            d = os.path.join(tmp, name)
            os.makedirs(os.path.join(d, "images"))
            os.makedirs(os.path.join(d, "labels"))
            files, sources = [], []
            for k, (h, w, nl) in enumerate(spec):
                img = synth_image(h, w, 1 if gray else 3, source_seed(name, k))
                f = os.path.join(d, "images", "%s_%02d.png" % (name, k))
                assert cv2.imwrite(f, img[:, :, 0] if gray else img)
                files.append(f)
                sources.append([h, w, 1 if gray else 3, source_seed(name, k)])
                if nl is not None:
                    with open(os.path.join(d, "labels", "%s_%02d.txt" % (name, k)), "w") as fh:
                        fh.write(synth_labels(nl, source_seed(name, k)))
            lst = os.path.join(d, "list.txt")
            with open(lst, "w") as fh:
                fh.write("\n".join(files) + "\n")
            ds = LoadImagesAndLabels(lst, s, bs, augment=True, hyp=hyp, rect=False, image_weights=iw,
                                     cache_images=cache, is_gray_scale=gray)
            assert [os.path.basename(f) for f in ds.img_files] == [os.path.basename(f) for f in files]
            torch.manual_seed(seed)
            random.seed(seed)
            np.random.seed(seed)
            indices = None
            if iw:                                 # train.py:334-337, once per epoch
                w = labels_to_image_weights(ds.labels, nc=80, class_weights=np.ones(80))
                ds.indices = random.choices(range(ds.n), weights=w, k=ds.n)
                indices = [int(i) for i in ds.indices]
            loader = torch.utils.data.DataLoader(ds, batch_size=bs, num_workers=0, shuffle=True,
                                                 collate_fn=ds.collate_fn)
            nb = 0
            for b, (imgs, targets, paths, shapes) in enumerate(itertools.islice(loader, keep)):
                assert all(sh is None for sh in shapes)
                out["%s_b%d_img" % (name, b)] = imgs.numpy()
                out["%s_b%d_targets" % (name, b)] = targets.numpy()
                out["%s_b%d_paths" % (name, b)] = np.array(json.dumps([os.path.basename(p) for p in paths]))
                print(name, b, tuple(imgs.shape), tuple(targets.shape), [os.path.basename(p) for p in paths])
                nb += 1
            rs = random.getstate()
            out[name + "_random_state"] = np.array(rs[1], np.uint64)
            ns = np.random.get_state()
            out[name + "_np_state"] = ns[1]
            out[name + "_np_pos"] = np.array(ns[2])
            out[name + "_torch_state"] = torch.get_rng_state().numpy()
            for i in range(len(ds.labels)):
                out["%s_labels%d" % (name, i)] = ds.labels[i]
            meta = dict(img_size=s, batch_size=bs, gray=gray, cache=cache, image_weights=iw, hyp=hyp, seed=seed,
                        files=[os.path.basename(f) for f in files], sources=sources, indices=indices, n_batches=nb,
                        epoch_batches=len(loader))
            out[name + "_meta"] = np.array(json.dumps(meta))
    finally:
        shutil.rmtree(tmp)
    path = os.path.join(ROOT, "tests", "golden", "trainloader_case.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
