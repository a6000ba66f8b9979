"""GPU: DeviceEvalLoader and b2y_load_batch_u8 (the device evaluation loader: load_image's INTER_AREA, the rect letterbox
border, the channel shuffle, one launch per batch) against the reference's own LoadImagesAndLabels(rect=True) +
collate_fn batches (tests/golden/evalloader_case.npz, oracle/gen_golden_evalloader.py).  Bit-exact."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from helpers import build_model
import evalloader_case as ec

pytestmark = pytest.mark.gpu


def _check(name, loader):
    m = ec.meta(name)
    assert len(loader) == m["n_batches"]
    n = 0
    for b, (imgs, targets, paths, shapes) in enumerate(loader):
        ref_img, ref_t, ref_paths, ref_shapes = ec.reference_batch(name, b)
        assert imgs.is_cuda and imgs.dtype == torch.uint8 and targets.is_cuda and targets.dtype == torch.float32
        got = imgs.cpu().numpy()
        assert got.shape == ref_img.shape, (name, b, got.shape, ref_img.shape)
        assert np.array_equal(got, ref_img), (name, b, int((got != ref_img).sum()))
        t = targets.cpu().numpy()
        assert t.shape == ref_t.shape and np.array_equal(t.view(np.uint32), ref_t.view(np.uint32)), (name, b)
        assert tuple(os.path.basename(p) for p in paths) == ref_paths
        assert shapes == ref_shapes
        n += 1
    assert n == m["n_batches"]


@pytest.mark.parametrize("name", ec.NAMES)
def test_batches_equal_reference(name, tmp_path):
    """Sources decoded from PNG files, as test.py's loader reads them."""
    pytest.importorskip("cv2")
    from b200yolo.preprocess import DeviceEvalLoader
    ds = ec.Dataset(name, directory=str(tmp_path))
    loader = DeviceEvalLoader(ds, ec.meta(name)["batch_size"])
    assert loader.dataset is ds
    _check(name, loader)


@pytest.mark.parametrize("name", ("c416", "c320"))
def test_cached_images_equal_reference(name):
    """--cache-images: the dataset holds load_image's outputs; the loader only pads and shuffles them."""
    pytest.importorskip("cv2")
    from b200yolo.preprocess import DeviceEvalLoader
    _check(name, DeviceEvalLoader(ec.Dataset(name, cache=True), ec.meta(name)["batch_size"]))


def test_one_launch_per_batch(tmp_path):
    """Every batch of mixed source sizes (block-mean, fractional and copied items together) is ONE kernel launch."""
    pytest.importorskip("cv2")
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from b200yolo.preprocess import DeviceEvalLoader
    loader = DeviceEvalLoader(ec.Dataset("c416", directory=str(tmp_path)), ec.meta("c416")["batch_size"])
    for b in range(len(loader)):
        plans = loader.host_batch(b)
        assert len({p["img"].shape for p in plans}) == len(plans)          # different source sizes in one batch
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            imgs = loader.device_batch(plans)[0]
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        kernels = [k for k in names if not k.startswith(("Memcpy", "Memset"))]
        assert len(kernels) == 1 and "load_batch_u8_kernel" in kernels[0], names
        assert np.array_equal(imgs.cpu().numpy(), ec.reference_batch("c416", b)[0])


def test_loader_batch_through_the_eval_engine(tmp_path):
    """A loader batch fed to the model gives the same io as the reference's bytes uploaded directly."""
    pytest.importorskip("cv2")
    from b200yolo.preprocess import DeviceEvalLoader
    model = build_model("yolov3-tiny", device="cuda").eval()
    loader = DeviceEvalLoader(ec.Dataset("c416", directory=str(tmp_path)), ec.meta("c416")["batch_size"])
    for b, (imgs, _, _, _) in enumerate(loader):
        with torch.no_grad():
            io = model(imgs)[0].clone()
            io_ref = model(torch.from_numpy(ec.reference_batch("c416", b)[0]).cuda())[0]
        assert torch.equal(io, io_ref), b


def test_refuses_what_it_does_not_build(tmp_path):
    from b200yolo.preprocess import DeviceEvalLoader
    ds = ec.Dataset("c320")
    ds.augment = True
    with pytest.raises(ValueError):
        DeviceEvalLoader(ds, 3)
    ds = ec.Dataset("c320")
    ds.rect = False
    with pytest.raises(ValueError):
        DeviceEvalLoader(ds, 3)
    # a batch shape smaller than the resized image: letterbox would resize a second time
    pytest.importorskip("cv2")
    ds = ec.Dataset("c320", directory=str(tmp_path))
    ds.batch_shapes = ds.batch_shapes // 2
    with pytest.raises(NotImplementedError, match=os.path.basename(ds.img_files[0])):
        DeviceEvalLoader(ds, 3).batch(0)


def test_c_abi_refuses_invalid_items():
    from b200yolo import lib
    from b200yolo.lib import LoadItem, call, ptr, stream_ptr
    src = torch.zeros((48, 64, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((1, 3, 32, 32), dtype=torch.uint8, device="cuda")
    good = dict(src=src.data_ptr(), src_pitch=64 * 3, src_h=48, src_w=64, rs_h=24, rs_w=32, area_kx=2, area_ky=2,
                scale_x=2.0, scale_y=2.0, top=4, left=0, slot=0)

    def run(**kw):
        items = (LoadItem * 1)(LoadItem(**dict(good, **kw)))
        dev = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
        call("b2y_load_batch_u8", C.cast(items, C.c_void_p), ptr(dev), 1, ptr(out), 1, 3, 32, 32, 1, 114, stream_ptr())

    run()
    torch.cuda.synchronize()
    for bad in (dict(src=None), dict(rs_h=30), dict(top=9), dict(left=-1), dict(slot=1), dict(area_kx=0, area_ky=0),
                dict(area_kx=3), dict(scale_x=2.0000001), dict(rs_w=65, scale_x=64 / 65), dict(src_pitch=100),
                dict(rs_w=30, scale_x=1.0 / (30 / 64))):
        with pytest.raises(lib.B2YError):
            run(**bad)
