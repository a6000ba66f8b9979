"""CPU: the evaluation loader's per-pixel INTER_AREA code (csrc/preprocess_core.h, shared by the CUDA kernel of
b2y_load_batch_u8 and this host harness) against cv2.resize(INTER_AREA), and its host-side logic (load_image's size,
OpenCV's choice of algorithm, the rect letterbox border, the label mapping) against the reference's own
LoadImagesAndLabels(rect=True) + collate_fn batches (tests/golden/evalloader_case.npz).  Bit-exact.  The GPU test
(tests/test_gpu_evalloader.py) runs the same batches through the kernel."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from helpers import PKG, ROOT
import evalloader_case as ec


@pytest.fixture(scope="module")
def host_lib():
    d = tempfile.mkdtemp(prefix="b2y_areahost_")
    so = os.path.join(d, "libareahost.so")
    src = os.path.join(ROOT, "tests", "host", "area_host.cpp")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(PKG, "csrc"), src, "-o", so],
                   check=True)
    lib = C.CDLL(so)
    lib.b2y_area_resize_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p]
    lib.b2y_load_slot_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                       C.c_int, C.c_int]
    return lib


def test_inter_area_matches_cv2_on_random_sizes(host_lib):
    """250 seeded (source, destination) size pairs, 1 and 3 channels, down-scaling only (what load_image asks for):
    exact 2x / 3x / 4x factors on one and on both axes, 1-pixel results, scales just above 1 and far above, and
    quantised images that make rounding ties common.  Both of OpenCV's INTER_AREA algorithms must be exercised."""
    cv2 = pytest.importorskip("cv2")
    from b200yolo.preprocess import inter_area_params
    rng = np.random.default_rng(2024)
    pairs = [(24, 832, 12, 416), (36, 1248, 12, 416), (1664, 32, 416, 8), (51, 832, 25, 416), (1000, 3, 416, 1),
             (3, 1000, 1, 416), (8, 8, 4, 4), (9, 9, 3, 3), (6, 9, 3, 3), (640, 480, 320, 240), (421, 420, 416, 415),
             (375, 500, 312, 416), (2, 2, 1, 1), (7, 1, 2, 1)]
    while len(pairs) < 250:
        h0, w0 = int(rng.integers(2, 600)), int(rng.integers(2, 600))
        if rng.random() < 0.35:                       # integer factors on one or both axes
            kx, ky = int(rng.integers(1, 5)), int(rng.integers(1, 5))
            h, w = max(1, h0 // ky), max(1, w0 // kx)
            h0, w0 = (h * ky, w * kx) if rng.random() < 0.7 else (h * ky + int(rng.integers(0, ky)), w * kx)
        else:
            h, w = int(rng.integers(1, h0 + 1)), int(rng.integers(1, w0 + 1))
        if (h, w) != (h0, w0):
            pairs.append((h0, w0, h, w))
    paths = {"block": 0, "fractional": 0}
    for k, (h0, w0, h, w) in enumerate(pairs):
        c = 1 if k % 3 == 2 else 3
        img = rng.integers(0, 256, (h0, w0, c), dtype=np.uint8)
        if k % 4 == 1:
            img = (img // 64 * 64 + 2).astype(np.uint8)          # few levels: many exact .5 ties
        ref = cv2.resize(img if c == 3 else img[:, :, 0], (w, h), interpolation=cv2.INTER_AREA).reshape(h, w, c)
        sx, sy, kx, ky = inter_area_params(h0, w0, h, w)
        paths["block" if kx else "fractional"] += 1
        out = np.zeros((h, w, c), np.uint8)
        host_lib.b2y_area_resize_host(img.ctypes.data, h0, w0, c, w0 * c, h, w, kx, ky, sx, sy, out.ctypes.data)
        assert np.array_equal(out, ref), ("INTER_AREA", (h0, w0), (h, w), c, (kx, ky), int((out != ref).sum()))
    print("INTER_AREA paths exercised:", paths)
    assert paths["block"] >= 40 and paths["fractional"] >= 100, paths


def test_inter_area_path_choice():
    from b200yolo.preprocess import inter_area_params
    assert inter_area_params(24, 832, 12, 416)[2:] == (2, 2)
    assert inter_area_params(1664, 32, 416, 8)[2:] == (4, 4)
    assert inter_area_params(51, 832, 25, 416)[2:] == (0, 0)        # x exact, y not: the fractional path
    assert inter_area_params(1664, 90, 416, 22)[2:] == (0, 0)


def _planned(name, tmp):
    from b200yolo.preprocess import DeviceEvalLoader
    m = ec.meta(name)
    return DeviceEvalLoader(ec.Dataset(name, directory=tmp), m["batch_size"]), m


@pytest.mark.parametrize("name", ec.NAMES)
def test_host_plan_and_pixels_match_reference(name, host_lib, tmp_path):
    """Every batch of the reference: sizes, border and shapes from the loader's host plan, the batch bytes from the
    kernel's per-pixel code run on the host, targets from the host label mapping -- all bit for bit."""
    pytest.importorskip("cv2")
    import torch
    loader, m = _planned(name, str(tmp_path))
    assert len(loader) == m["n_batches"]
    for b in range(len(loader)):
        ref_img, ref_t, ref_paths, ref_shapes = ec.reference_batch(name, b)
        plans = loader.host_batch(b)
        B, cn, H, W = ref_img.shape
        got = np.zeros_like(ref_img)
        for k, p in enumerate(plans):
            img = p["img"]
            assert p["out"] == (H, W) and img.shape[2] == cn
            sx, sy, kx, ky = p["scales"]
            host_lib.b2y_load_slot_host(img.ctypes.data, img.shape[0], img.shape[1], cn, img.shape[1] * cn,
                                        p["rs"][0], p["rs"][1], kx, ky, sx, sy, p["top"], p["left"],
                                        got[k].ctypes.data, H, W, 1 if cn == 3 else 0, 114)
        assert np.array_equal(got, ref_img), (name, b, int((got != ref_img).sum()))
        targets = torch.cat([torch.cat([torch.full((len(p["labels"]), 1), float(k)),
                                        torch.from_numpy(p["labels"])], 1) for k, p in enumerate(plans)], 0)
        assert targets.dtype == torch.float32
        assert np.array_equal(targets.numpy().view(np.uint32), ref_t.view(np.uint32)), (name, b)
        assert tuple(os.path.basename(p["path"]) for p in plans) == ref_paths
        assert tuple(p["shapes"] for p in plans) == ref_shapes


def test_fixture_covers_the_cases():
    """Both INTER_AREA paths, copies, 1-pixel results, images without labels, two image sizes, gray-scale."""
    from b200yolo.preprocess import inter_area_params, load_image_size
    kinds, one_px, sizes, empty = set(), False, set(), 0
    for name in ec.NAMES:
        m = ec.meta(name)
        sizes.add(m["img_size"])
        for (h0, w0, c, _), lab in zip(m["sources"], ec.Dataset(name).labels):
            h, w = load_image_size(h0, w0, m["img_size"])
            one_px |= min(h, w) == 1
            empty += lab.size == 0
            kinds.add("copy" if (h, w) == (h0, w0) else ("block" if inter_area_params(h0, w0, h, w)[2] else "frac"))
    assert kinds == {"copy", "block", "frac"} and one_px and sizes == {320, 416} and empty >= 2
    assert any(ec.meta(n)["gray"] for n in ec.NAMES)
