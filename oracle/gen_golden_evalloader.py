"""Generate tests/golden/evalloader_case.npz by RUNNING THE REFERENCE's evaluation loader: LoadImagesAndLabels(rect=True)
(utils/datasets.py:262-475, 511-531: cv2.imread, load_image's INTER_AREA downscale, the rect letterbox, the label mapping)
and its collate_fn, over seeded synthetic datasets written to a temporary directory as PNG (lossless, so decoding is not
a variable).  Stores, per dataset and in the dataset's (aspect-sorted) order, the file names, the source sizes and
seeds (preprocess_oracle.synth_image regenerates the decoded sources: integer arithmetic only, checked here against
cv2.imread of the PNGs), the parsed labels; its batch index and batch shapes; and every batch's image bytes, targets,
paths (file names) and shapes.  Run where the reference is (the GPU machines have none); the output is committed.

    python oracle/gen_golden_evalloader.py
"""
import json
import os
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

sys.path.insert(0, HERE)
from preprocess_oracle import synth_image  # noqa: E402

# name, img_size, batch_size, gray, [(h0, w0, n_labels or None = no label file)]
DATASETS = [
    ("c416", 416, 4, False, [
        (24, 832, 2),       # 2x on both axes -> 12 x 416 (block mean, 2 x 2 rounding)
        (36, 1248, 1),      # 3x on both axes -> 12 x 416
        (1664, 32, 3),      # 4x on both axes -> 416 x 8
        (51, 832, 2),       # 2x on x, fractional on y -> 25 x 416
        (1248, 50, 0),      # 3x on y, fractional on x -> 416 x 16; empty label file
        (1664, 90, 2),      # 4x on y, fractional on x -> 416 x 22
        (1000, 3, 1),       # 1-pixel-wide result -> 416 x 1
        (450, 120, 4),      # fractional, scale close to 1.08 -> 416 x 110
        (100, 300, 2),      # smaller than img_size: copy + border
        (200, 50, None),    # smaller, no label file
        (430, 200, 3),      # fractional -> 416 x 193
        (60, 420, 1),       # barely larger: scale 1.0096 -> 59 x 416
    ]),
    ("c320", 320, 3, False, [
        (640, 64, 2),       # 2x both -> 320 x 32
        (960, 40, 1),       # 3x on y, fractional on x -> 320 x 13
        (400, 100, 3),      # fractional 1.25 both -> 320 x 80
        (20, 700, 1),       # -> 9 x 320
        (321, 321, 5),      # scale 1.003 -> 320 x 320
        (48, 1280, 2),      # 4x both -> 12 x 320
        (50, 1280, None),   # 4x on x, fractional on y -> 12 x 320
        (330, 30, 2),       # -> 320 x 29
        (100, 200, 1),      # smaller
    ]),
    ("g320", 320, 2, True, [
        (640, 32, 2),       # 2x both -> 320 x 16
        (100, 700, 1),      # fractional -> 45 x 320
        (30, 200, 2),       # smaller
        (960, 96, 0),       # 3x both -> 320 x 32
    ]),
]


def synth_labels(n, seed):
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n):
        w, h = rng.uniform(0.02, 0.6), rng.uniform(0.02, 0.6)
        x, y = rng.uniform(w / 2, 1 - w / 2), rng.uniform(h / 2, 1 - h / 2)
        rows.append("%d %.6f %.6f %.6f %.6f" % (rng.integers(0, 80), x, y, w, h))
    return "\n".join(rows) + ("\n" if rows else "")


def source_seed(name, img_size, k):
    return 1000 * len(name) + 17 * k + img_size


def run_dataset(name, img_size, bs, gray, spec, tmp, cache):
    from utils.datasets import LoadImagesAndLabels
    d = os.path.join(tmp, name + ("_cache" if cache else ""))
    os.makedirs(os.path.join(d, "images"))
    os.makedirs(os.path.join(d, "labels"))
    files = []
    for k, (h, w, nl) in enumerate(spec):
        seed = source_seed(name, img_size, k)
        img = synth_image(h, w, 1 if gray else 3, seed)
        f = os.path.join(d, "images", "%s_%02d.png" % (name, k))
        assert cv2.imwrite(f, img[:, :, 0] if gray else img)
        files.append(f)
        if nl is not None:
            with open(os.path.join(d, "labels", "%s_%02d.txt" % (name, k)), "w") as fh:
                fh.write(synth_labels(nl, seed))
    lst = os.path.join(d, "list.txt")
    with open(lst, "w") as fh:
        fh.write("\n".join(files) + "\n")
    ds = LoadImagesAndLabels(lst, img_size, bs, augment=False, rect=True, cache_images=cache, is_gray_scale=gray)
    batches = []
    for b0 in range(0, len(ds), bs):
        batches.append(ds.collate_fn([ds[i] for i in range(b0, min(len(ds), b0 + bs))]))
    return ds, batches


def main():
    os.chdir(REF)
    np.int = int                               # datasets.py:278 still uses the alias removed from numpy
    out = {}
    tmp = tempfile.mkdtemp(prefix="b2y_evalloader_")
    try:
        for name, img_size, bs, gray, spec in DATASETS:
            ds, batches = run_dataset(name, img_size, bs, gray, spec, tmp, False)
            if not gray:       # the --cache-images path gives the same batches
                _, cb = run_dataset(name, img_size, bs, gray, spec, tmp, True)
                for a, c in zip(batches, cb):
                    assert np.array_equal(a[0].numpy(), c[0].numpy()) and np.array_equal(a[1].numpy(), c[1].numpy())
            files = [os.path.basename(f) for f in ds.img_files]
            sources = []
            for i, f in enumerate(ds.img_files):
                k = int(files[i][len(name) + 1:-4])
                h, w, _ = spec[k]
                img = cv2.imread(f, cv2.IMREAD_GRAYSCALE) if gray else cv2.imread(f)
                assert np.array_equal(img.reshape(h, w, -1), synth_image(h, w, 1 if gray else 3,
                                                                         source_seed(name, img_size, k)))
                sources.append([h, w, 1 if gray else 3, source_seed(name, img_size, k)])
                out["%s_labels%d" % (name, i)] = ds.labels[i]
            meta = dict(img_size=img_size, batch_size=bs, gray=gray, files=files, sources=sources,
                        batch=[int(v) for v in ds.batch], batch_shapes=[[int(v) for v in s] for s in ds.batch_shapes],
                        n_batches=len(batches))
            out[name + "_meta"] = np.array(json.dumps(meta))
            for b, (imgs, targets, paths, shapes) in enumerate(batches):
                out["%s_b%d_img" % (name, b)] = imgs.numpy()
                out["%s_b%d_targets" % (name, b)] = targets.numpy()
                out["%s_b%d_paths" % (name, b)] = np.array(json.dumps([os.path.basename(p) for p in paths]))
                out["%s_b%d_shapes" % (name, b)] = np.array(json.dumps(shapes))
                print(name, b, tuple(imgs.shape), tuple(targets.shape), [os.path.basename(p) for p in paths])
    finally:
        shutil.rmtree(tmp)
    path = os.path.join(ROOT, "tests", "golden", "evalloader_case.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
