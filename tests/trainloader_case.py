"""The training-loader datasets of tests/golden/trainloader_case.npz (oracle/gen_golden_trainloader.py: the reference's
LoadImagesAndLabels(augment=True) under a seeded num_workers=0 DataLoader(shuffle=True, collate_fn) over seeded PNG
datasets), rebuilt as duck-typed datasets with the reference's attributes, and the reference's batches and RNG states.
The fixture keeps the first n_batches batches of each epoch and the RNG states after them."""
import json
import os
import random
import sys

import numpy as np

from helpers import ROOT, golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
from preprocess_oracle import synth_image  # noqa: E402

NAMES = ("c128", "c128u", "c160", "c160w", "g128")
_G = None


def fixture():
    global _G
    if _G is None:
        _G = golden("trainloader_case")
    return _G


def meta(name):
    return json.loads(str(fixture()[name + "_meta"]))


class Dataset:
    """The attributes of LoadImagesAndLabels(augment=True, rect=False) that the training loader reads.  With the
    fixture's cache flag, imgs / img_hw0 / img_hw hold load_image's outputs (cv2.resize INTER_LINEAR), as
    --cache-images keeps them; otherwise the sources are written as PNG files under `directory`."""

    def __init__(self, name, directory=None):
        m = meta(name)
        g = fixture()
        n = len(m["files"])
        self.n = n
        self.img_size, self.is_gray_scale, self.hyp = m["img_size"], m["gray"], m["hyp"]
        self.augment, self.rect, self.image_weights = True, False, m["image_weights"]
        if m["indices"] is not None:
            self.indices = m["indices"]
        self.labels = [g["%s_labels%d" % (name, i)] for i in range(n)]
        self.img_files = [os.path.join(directory or "", f) for f in m["files"]]
        self.imgs = [None] * n
        srcs = [synth_image(h, w, c, seed) for h, w, c, seed in m["sources"]]
        import cv2
        if m["cache"]:
            from b200yolo.preprocess import train_tile_size
            self.img_hw0, self.img_hw = [], []
            for i, s in enumerate(srcs):
                h0, w0 = s.shape[:2]
                h, w = train_tile_size(h0, w0, self.img_size)
                if (h, w) != (h0, w0):
                    s = cv2.resize(s, (w, h), interpolation=cv2.INTER_LINEAR).reshape(h, w, -1)
                self.imgs[i] = s
                self.img_hw0.append((h0, w0))
                self.img_hw.append((h, w))
        else:
            assert directory is not None, name + " reads its sources from files"
            for f, s in zip(self.img_files, srcs):
                assert cv2.imwrite(f, s[:, :, 0] if self.is_gray_scale else s)

    def __len__(self):
        return self.n


def seed(name):
    """The seeds the fixture's epoch started from; an image_weights epoch first makes train.py's random.choices draw
    (its indices are in the fixture)."""
    import torch
    m = meta(name)
    torch.manual_seed(m["seed"])
    random.seed(m["seed"])
    np.random.seed(m["seed"])
    if m["indices"] is not None:
        random.choices(range(len(m["files"])), weights=[1.0] * len(m["files"]), k=len(m["files"]))


def fixture_labels(name):
    g = fixture()
    return [g["%s_labels%d" % (name, i)] for i in range(len(meta(name)["files"]))]


def reference_batch(name, b):
    """(uint8 images, float32 targets, file names) of the reference's batch b."""
    g = fixture()
    return (g["%s_b%d_img" % (name, b)], g["%s_b%d_targets" % (name, b)],
            tuple(json.loads(str(g["%s_b%d_paths" % (name, b)]))))


def rng_states_equal(name):
    """The random, np.random and torch CPU generator states equal the reference's after the batches the fixture
    keeps (the first n_batches of an epoch of epoch_batches)."""
    import torch
    g = fixture()
    return (np.array_equal(np.array(random.getstate()[1], np.uint64), g[name + "_random_state"]) and
            np.array_equal(np.random.get_state()[1], g[name + "_np_state"]) and
            int(np.random.get_state()[2]) == int(g[name + "_np_pos"]) and
            np.array_equal(torch.get_rng_state().numpy(), g[name + "_torch_state"]))
