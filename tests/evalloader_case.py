"""The evaluation-loader datasets of tests/golden/evalloader_case.npz (oracle/gen_golden_evalloader.py: the reference's
LoadImagesAndLabels(rect=True) + collate_fn over seeded PNG datasets), rebuilt as duck-typed datasets with the
reference's attributes, and the reference's batches."""
import json
import os
import sys

import numpy as np

from helpers import ROOT, golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
from preprocess_oracle import synth_image  # noqa: E402

NAMES = ("c416", "c320", "g320")
_G = None


def fixture():
    global _G
    if _G is None:
        _G = golden("evalloader_case")
    return _G


def meta(name):
    return json.loads(str(fixture()[name + "_meta"]))


def sources(name):
    """Decoded sources in the dataset's order: HWC uint8 (gray-scale: [h, w, 1])."""
    return [synth_image(h, w, c, seed) for h, w, c, seed in meta(name)["sources"]]


class Dataset:
    """The attributes of LoadImagesAndLabels(rect=True, augment=False) that evaluation loading reads."""

    def __init__(self, name, directory=None, cache=False):
        m = meta(name)
        g = fixture()
        n = len(m["files"])
        self.img_size, self.is_gray_scale, self.augment, self.rect = m["img_size"], m["gray"], False, True
        self.batch = np.array(m["batch"])
        self.batch_shapes = np.array(m["batch_shapes"])
        self.labels = [g["%s_labels%d" % (name, i)] for i in range(n)]
        self.img_files = [os.path.join(directory or "", f) for f in m["files"]]
        self.imgs = [None] * n
        srcs = sources(name)
        if directory is not None:
            import cv2
            for f, s in zip(self.img_files, srcs):
                assert cv2.imwrite(f, s[:, :, 0] if self.is_gray_scale else s)
        if cache:                          # load_image's outputs, as --cache-images keeps them
            import cv2
            from b200yolo.preprocess import load_image_size
            self.img_hw0, self.img_hw = [], []
            for i, s in enumerate(srcs):
                h0, w0 = s.shape[:2]
                h, w = load_image_size(h0, w0, self.img_size)
                if (h, w) != (h0, w0):
                    s = cv2.resize(s, (w, h), interpolation=cv2.INTER_AREA).reshape(h, w, -1)
                self.imgs[i] = s
                self.img_hw0.append((h0, w0))
                self.img_hw.append((h, w))

    def __len__(self):
        return len(self.img_files)


def reference_batch(name, b):
    """(uint8 images, float32 targets, file names, shapes) of the reference's batch b."""
    g = fixture()
    shapes = json.loads(str(g["%s_b%d_shapes" % (name, b)]))
    shapes = tuple(((s[0][0], s[0][1]), ((s[1][0][0], s[1][0][1]), (s[1][1][0], s[1][1][1]))) for s in shapes)
    return (g["%s_b%d_img" % (name, b)], g["%s_b%d_targets" % (name, b)],
            tuple(json.loads(str(g["%s_b%d_paths" % (name, b)]))), shapes)
