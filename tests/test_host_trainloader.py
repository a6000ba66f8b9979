"""CPU: the training loader's per-pixel code (csrc/preprocess_core.h, shared by the CUDA kernels of b2y_mosaic_u8 and
b2y_affine_hsv_u8 and this host harness) against cv2 -- BGR2HSV and HSV2BGR over every input, warpAffine on seeded
matrices, load_image's INTER_LINEAR tiles -- and its host plan (draw order, tiles, rectangles, affine map, LUTs,
labels, flips) plus the host-compiled pixels against the reference's own LoadImagesAndLabels(augment=True) batches
(tests/golden/trainloader_case.npz).  Bit-exact.  The GPU test (tests/test_gpu_trainloader.py) runs the same batches
through the kernels."""
import ctypes as C
import itertools
import math
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

from helpers import PKG, ROOT
import trainloader_case as tc

vp, i32, ll = C.c_void_p, C.c_int, C.c_longlong


@pytest.fixture(scope="module")
def host_lib():
    d = tempfile.mkdtemp(prefix="b2y_augmenthost_")
    so = os.path.join(d, "libaugmenthost.so")
    src = os.path.join(ROOT, "tests", "host", "augment_host.cpp")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(PKG, "csrc"), src, "-o", so],
                   check=True)
    lib = C.CDLL(so)
    lib.b2y_bgr2hsv_host.argtypes = [vp, vp, ll]
    lib.b2y_hsv2bgr_host.argtypes = [vp, vp, ll]
    lib.b2y_warp_host.argtypes = [vp, i32, i32, i32, vp, vp, i32, i32, i32]
    lib.b2y_tile_host.argtypes = [vp, i32, i32, i32, i32, i32, vp]
    lib.b2y_augment_slot_host.argtypes = [vp, i32, i32, i32, vp, vp, i32, vp, i32]
    return lib


def test_bgr2hsv_every_input(host_lib):
    cv2 = pytest.importorskip("cv2")
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)
    out = np.empty_like(img)
    host_lib.b2y_bgr2hsv_host(img.ctypes.data, out.ctypes.data, img.size // 3)
    ref = cv2.cvtColor(img, cv2.COLOR_BGR2HSV)
    assert np.array_equal(out, ref), int((out != ref).sum())


def test_hsv2bgr_every_input_default_dispatch(host_lib):
    """All 180 x 256 x 256 HSV triples in rows of 256 pixels, with cv2's default (optimised) dispatch, which the
    reference runs."""
    cv2 = pytest.importorskip("cv2")
    assert cv2.useOptimized()
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    img = np.stack([h, s, v], -1).astype(np.uint8).reshape(180 * 256, 256, 3)
    out = np.empty_like(img)
    host_lib.b2y_hsv2bgr_host(img.ctypes.data, out.ctypes.data, img.size // 3)
    ref = cv2.cvtColor(img, cv2.COLOR_HSV2BGR)
    assert np.array_equal(out, ref), int((out != ref).sum())


def test_hsv2bgr_training_row_widths(host_lib):
    """Random HSV images at the row widths of training batches (multiples of 32) agree with cv2 as whole images."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for w in (128, 160, 416, 640):
        img = np.stack([rng.integers(0, 180, (64, w)), rng.integers(0, 256, (64, w)), rng.integers(0, 256, (64, w))],
                       -1).astype(np.uint8)
        out = np.empty_like(img)
        host_lib.b2y_hsv2bgr_host(img.ctypes.data, out.ctypes.data, img.size // 3)
        assert np.array_equal(out, cv2.cvtColor(img, cv2.COLOR_HSV2BGR)), w


def _affine(s, a, sc, tx, ty, shx, shy):
    import cv2
    R = np.eye(3)
    R[:2] = cv2.getRotationMatrix2D(angle=a, center=(s, s), scale=sc)
    T = np.eye(3)
    T[0, 2], T[1, 2] = tx * 2 * s - s // 2, ty * 2 * s - s // 2
    S = np.eye(3)
    S[0, 1], S[1, 0] = math.tan(shx * math.pi / 180), math.tan(shy * math.pi / 180)
    return S @ T @ R


def test_warp_affine_matches_cv2(host_lib):
    """300 seeded cases: matrices drawn as random_affine draws them (with wider ranges, so taps leave the canvas),
    pure translations (train.py's default hyp), 1 and 3 channels."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    r = random.Random(7)
    kinds = {"general": 0, "translation": 0}
    for k in range(300):
        s = int(rng.choice([32, 64, 96, 128, 160]))
        c = 1 if k % 4 == 3 else 3
        src = rng.integers(0, 256, (2 * s, 2 * s, c), dtype=np.uint8)
        if k % 3 == 0:
            M = _affine(s, 0, 1, int(rng.integers(-s, s)) / (2 * s) if k % 2 else 0, 0, 0, 0)
            kinds["translation"] += 1
        else:
            M = _affine(s, r.uniform(-30, 30), r.uniform(0.7, 1.3), r.uniform(-.2, .2), r.uniform(-.2, .2),
                        r.uniform(-15, 15), r.uniform(-15, 15))
            kinds["general"] += 1
        ref = cv2.warpAffine(src, M[:2], dsize=(s, s), flags=cv2.INTER_LINEAR,
                             borderValue=(114, 114, 114)).reshape(s, s, c)
        im = np.ascontiguousarray(cv2.invertAffineTransform(M[:2]).reshape(-1))
        out = np.empty((s, s, c), np.uint8)
        host_lib.b2y_warp_host(src.ctypes.data, 2 * s, 2 * s, c, im.ctypes.data, out.ctypes.data, s, s, 114)
        assert np.array_equal(out, ref), (k, s, c, int((out != ref).sum()))
    assert min(kinds.values()) >= 90, kinds


def test_tile_resize_matches_cv2(host_lib):
    """load_image's INTER_LINEAR (augment=True: up and down), including cv::resize's exact-2x case, which it computes
    as the INTER_AREA 2 x 2 mean: the bilinear code gives the same bytes there."""
    cv2 = pytest.importorskip("cv2")
    from b200yolo.preprocess import train_tile_size
    rng = np.random.default_rng(9)
    sizes = [(1280, 1280, 640), (1280, 960, 640), (256, 192, 128), (60, 90, 128), (300, 3, 128), (2, 300, 160)]
    while len(sizes) < 150:
        sizes.append((int(rng.integers(2, 700)), int(rng.integers(2, 700)), int(rng.choice([128, 160, 320]))))
    for k, (h0, w0, s) in enumerate(sizes):
        h, w = train_tile_size(h0, w0, s)
        if min(h, w) < 1 or (h, w) == (h0, w0):
            continue
        c = 1 if k % 3 == 2 else 3
        src = rng.integers(0, 256, (h0, w0, c), dtype=np.uint8)
        ref = cv2.resize(src, (w, h), interpolation=cv2.INTER_LINEAR).reshape(h, w, c)
        if 2 * h == h0 and 2 * w == w0:
            assert np.array_equal(ref, cv2.resize(src, (w, h), interpolation=cv2.INTER_AREA).reshape(h, w, c))
        out = np.empty((h, w, c), np.uint8)
        host_lib.b2y_tile_host(src.ctypes.data, h0, w0, c, h, w, out.ctypes.data)
        assert np.array_equal(out, ref), ((h0, w0), (h, w), c, int((out != ref).sum()))


def host_canvas(host_lib, sources, plan, s):
    """load_mosaic's canvas as numpy builds it: 114, then each tile's slice assigned in tile order."""
    cn = next(iter(sources.values()))[0].shape[2]
    canvas = np.full((2 * s, 2 * s, cn), 114, np.uint8)
    for i, ((x1a, y1a, x2a, y2a), (dx, dy)) in zip(plan["tiles"], plan["rects"]):
        img, (h, w) = sources[i]
        if (h, w) != img.shape[:2]:
            tile = np.empty((h, w, cn), np.uint8)
            host_lib.b2y_tile_host(img.ctypes.data, img.shape[0], img.shape[1], cn, h, w, tile.ctypes.data)
        else:
            tile = img
        canvas[y1a:y2a, x1a:x2a] = tile[y1a + dy:y2a + dy, x1a + dx:x2a + dx]
    return canvas


@pytest.mark.parametrize("name", tc.NAMES)
def test_host_plan_and_pixels_match_reference(name, host_lib, tmp_path):
    """Every batch the fixture keeps of the reference's epoch: index order, draws, tiles, rectangles, affine map, LUTs and flips from the
    loader's host plan, the batch bytes from the kernels' per-pixel code run on the host over a numpy mosaic, targets
    from the host label mapping -- bit for bit -- and the three RNG states after those batches."""
    pytest.importorskip("cv2")
    import torch
    from b200yolo.preprocess import DeviceTrainLoader
    m = tc.meta(name)
    s = m["img_size"]
    loader = DeviceTrainLoader(tc.Dataset(name, directory=str(tmp_path)), m["batch_size"])
    assert len(loader) == m["epoch_batches"]
    tc.seed(name)
    n = 0
    for b, indices in enumerate(itertools.islice(loader._index, m["n_batches"])):
        ref_img, ref_t, ref_paths = tc.reference_batch(name, b)
        sources, plans = loader.host_batch(indices)
        got = np.zeros_like(ref_img)
        for k, p in enumerate(plans):
            canvas = host_canvas(host_lib, sources, p, s)
            im = np.ascontiguousarray(p["im"].reshape(-1))
            lut = None if p["lut"] is None else np.ascontiguousarray(p["lut"])
            host_lib.b2y_augment_slot_host(canvas.ctypes.data, 2 * s, 2 * s, canvas.shape[2], im.ctypes.data,
                                           None if lut is None else lut.ctypes.data, int(p["flip"]), got[k].ctypes.data, s)
        assert np.array_equal(got, ref_img), (name, b, int((got != ref_img).sum()))
        targets = torch.cat([torch.cat([torch.full((len(p["labels"]), 1), float(k)), torch.from_numpy(p["labels"])], 1)
                             for k, p in enumerate(plans)], 0)
        assert targets.dtype == torch.float32
        assert np.array_equal(targets.numpy().view(np.uint32), ref_t.view(np.uint32)), (name, b)
        assert tuple(os.path.basename(p["path"]) for p in plans) == ref_paths
        n += 1
    assert n == m["n_batches"]
    assert tc.rng_states_equal(name)


def test_fixture_covers_the_cases():
    """Both image sizes, colour and gray-scale, cached and uncached, an image_weights epoch, both hyp sets; sources
    larger (fractional and exact 2x), smaller, equal and 1 pixel thin; an empty label file; boxes the affine drops."""
    from b200yolo.preprocess import train_tile_size
    kinds, thin, sizes, empty = set(), False, set(), 0
    for name in tc.NAMES:
        m = tc.meta(name)
        sizes.add(m["img_size"])
        for (h0, w0, _, _), lab in zip(m["sources"], tc.fixture_labels(name)):
            h, w = train_tile_size(h0, w0, m["img_size"])
            thin |= min(h, w) == 1
            empty += lab.size == 0
            kinds.add("equal" if (h, w) == (h0, w0) else ("2x" if (2 * h, 2 * w) == (h0, w0) else
                                                           ("up" if h > h0 else "down")))
    assert kinds == {"equal", "2x", "up", "down"} and thin and sizes == {128, 160} and empty >= 2
    metas = [tc.meta(n) for n in tc.NAMES]
    assert any(m["gray"] for m in metas) and any(m["cache"] for m in metas) and any(not m["cache"] for m in metas)
    assert any(m["image_weights"] for m in metas)
    assert {m["hyp"]["degrees"] for m in metas} == {0, 10}
    # some box of the reference's labels does not survive: fewer targets than mosaic boxes somewhere
    dropped = False
    for name in tc.NAMES:
        for b in range(tc.meta(name)["n_batches"]):
            dropped |= len(tc.reference_batch(name, b)[1]) < 4 * tc.meta(name)["batch_size"]
    assert dropped


def test_refuses_what_it_does_not_build():
    from b200yolo.preprocess import DeviceTrainLoader
    ds = tc.Dataset("c128")
    ds.augment = False
    with pytest.raises(ValueError, match="DeviceEvalLoader"):
        DeviceTrainLoader(ds, 4)
    ds = tc.Dataset("c128")
    ds.rect = True
    with pytest.raises(ValueError, match="rect"):
        DeviceTrainLoader(ds, 4)
