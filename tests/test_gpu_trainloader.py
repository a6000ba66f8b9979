"""GPU: DeviceTrainLoader, b2y_mosaic_u8 and b2y_affine_hsv_u8 (the device training loader: mosaic, random affine, HSV,
flip and channel shuffle, two launches per batch) against the reference's own LoadImagesAndLabels(augment=True) +
num_workers=0 DataLoader batches (tests/golden/trainloader_case.npz, oracle/gen_golden_trainloader.py).  Bit-exact."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch

from helpers import attach_hyp, build_model
import trainloader_case as tc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", tc.NAMES)
def test_batches_equal_reference(name, tmp_path):
    pytest.importorskip("cv2")
    from b200yolo.preprocess import DeviceTrainLoader
    m = tc.meta(name)
    ds = tc.Dataset(name, directory=str(tmp_path))
    loader = DeviceTrainLoader(ds, m["batch_size"])
    assert loader.dataset is ds and len(loader) == m["epoch_batches"]
    tc.seed(name)
    n = 0
    for b, (imgs, targets, paths, shapes) in enumerate(itertools.islice(loader, m["n_batches"])):
        ref_img, ref_t, ref_paths = tc.reference_batch(name, b)
        assert imgs.is_cuda and imgs.dtype == torch.uint8 and targets.is_cuda and targets.dtype == torch.float32
        got = imgs.cpu().numpy()
        assert got.shape == ref_img.shape, (name, b, got.shape, ref_img.shape)
        assert np.array_equal(got, ref_img), (name, b, int((got != ref_img).sum()))
        t = targets.cpu().numpy()
        assert t.shape == ref_t.shape and np.array_equal(t.view(np.uint32), ref_t.view(np.uint32)), (name, b)
        assert tuple(os.path.basename(p) for p in paths) == ref_paths
        assert shapes == (None,) * len(paths)
        n += 1
    assert n == m["n_batches"]
    assert tc.rng_states_equal(name)


def test_distributed_sampler_drives_the_order():
    """A DistributedSampler given as `sampler` is what `.sampler` returns, and set_epoch changes the order."""
    pytest.importorskip("cv2")
    from b200yolo.preprocess import DeviceTrainLoader
    ds = tc.Dataset("c160")
    sampler = torch.utils.data.distributed.DistributedSampler(ds, num_replicas=2, rank=1, shuffle=True, seed=3)
    loader = DeviceTrainLoader(ds, 2, shuffle=False, sampler=sampler)
    assert loader.sampler is sampler and len(loader) == 2
    orders = []
    for epoch in (0, 1):
        loader.sampler.set_epoch(epoch)
        orders.append([list(i) for i in loader._index])
        paths = next(iter(loader))[2]
        assert list(paths) == [ds.img_files[i] for i in orders[-1][0]]
    assert orders[0] != orders[1]


def _profile_launches(directory):
    """Profile the device stage of every c128u batch; returns, per batch, the names of the CUDA kernels launched and
    whether the bytes equal the reference's."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from b200yolo.preprocess import DeviceTrainLoader
    loader = DeviceTrainLoader(tc.Dataset("c128u", directory=directory), tc.meta("c128u")["batch_size"])
    tc.seed("c128u")
    out = []
    for b, indices in enumerate(itertools.islice(loader._index, tc.meta("c128u")["n_batches"])):
        planned = loader.host_batch(indices)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            imgs = loader.device_batch(planned)[0]
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        out.append(([k for k in names if not k.startswith(("Memcpy", "Memset"))],
                    bool(np.array_equal(imgs.cpu().numpy(), tc.reference_batch("c128u", b)[0]))))
    return out


def test_two_launches_per_batch(tmp_path):
    """Every batch is two C-ABI calls, b2y_mosaic_u8 then b2y_affine_hsv_u8, and two kernels on the device.  The
    profiler runs in a process of its own: in a long pytest process, state left by earlier CUDA work can make a later
    profiler session report no device activity at all."""
    pytest.importorskip("cv2")
    import json
    import subprocess
    import sys
    from helpers import PKG, ROOT
    from b200yolo import lib
    from b200yolo.preprocess import DeviceTrainLoader
    loader = DeviceTrainLoader(tc.Dataset("c128u", directory=str(tmp_path)), tc.meta("c128u")["batch_size"])
    tc.seed("c128u")
    for indices in itertools.islice(loader._index, tc.meta("c128u")["n_batches"]):
        planned = loader.host_batch(indices)
        lib.RECORD = []
        try:
            loader.device_batch(planned)
            calls = [name for name, _ in lib.RECORD]
        finally:
            lib.RECORD = None
            lib.KEEPALIVE.clear()
        assert calls == ["b2y_mosaic_u8", "b2y_affine_hsv_u8"], calls
    code = ("import json, sys; sys.path[:0] = %r; import test_gpu_trainloader as t; "
            "print(json.dumps(t._profile_launches(%r)))" % ([os.path.join(ROOT, "tests"), PKG, ROOT],
                                                            str(tmp_path / "sub")))
    os.makedirs(tmp_path / "sub")
    run = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    batches = json.loads(run.stdout.strip().splitlines()[-1])
    assert len(batches) == tc.meta("c128u")["n_batches"]
    for kernels, same in batches:
        assert len(kernels) == 2 and "mosaic_u8_kernel" in kernels[0] and "affine_hsv_u8_kernel" in kernels[1], kernels
        assert same


def test_loader_batch_through_the_training_engine():
    """A loader batch through the training forward and compute_loss gives the loss of the reference's batch tensor."""
    pytest.importorskip("cv2")
    from utils import utils as my_utils
    from b200yolo.preprocess import DeviceTrainLoader
    model = attach_hyp(build_model("yolov3-tiny", device="cuda")).train()
    loader = DeviceTrainLoader(tc.Dataset("c128"), tc.meta("c128")["batch_size"])
    tc.seed("c128")
    imgs, targets, _, _ = next(iter(loader))
    ref_img, ref_t, _ = tc.reference_batch("c128", 0)
    pred, _ = model(imgs)
    loss, items = my_utils.compute_loss(pred, targets, model)
    pred_ref, _ = model(torch.from_numpy(ref_img).cuda())
    loss_ref, items_ref = my_utils.compute_loss(pred_ref, torch.from_numpy(ref_t).cuda(), model)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all() and torch.equal(loss, loss_ref) and torch.equal(items, items_ref)


def test_c_abi_refuses_invalid_items():
    from b200yolo import lib
    from b200yolo.lib import AffineItem, MosaicItem, MosaicTile, call, ptr, stream_ptr
    s = 32
    src = torch.zeros((40, 50, 3), dtype=torch.uint8, device="cuda")
    canvas = torch.empty((1, 2 * s, 2 * s, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((1, 3, s, s), dtype=torch.uint8, device="cuda")
    tile = dict(src=src.data_ptr(), src_pitch=50 * 3, src_h=40, src_w=50, rs_h=20, rs_w=25, scale_x=2.0, scale_y=2.0,
                x1a=0, y1a=0, x2a=25, y2a=20, dx=0, dy=0)

    def mosaic(**kw):
        item = MosaicItem()
        for k in range(4):
            item.tiles[k] = MosaicTile(**dict(tile, **kw))
        items = (MosaicItem * 1)(item)
        dev = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
        call("b2y_mosaic_u8", C.cast(items, C.c_void_p), ptr(dev), 1, ptr(canvas), 1, 3, s, stream_ptr())

    def affine(channels=3, **kw):
        item = AffineItem()
        item.im[:] = kw.pop("im", [1.0, 0.0, 16.0, 0.0, 1.0, 16.0])
        for k, v in kw.items():
            setattr(item, k, v)
        items = (AffineItem * 1)(item)
        dev = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
        call("b2y_affine_hsv_u8", C.cast(items, C.c_void_p), ptr(dev), 1, ptr(canvas), ptr(out), 1, channels, s,
             stream_ptr())

    mosaic()
    affine(hsv=1, flip=1)
    torch.cuda.synchronize()
    for bad in (dict(src=None), dict(src_pitch=100), dict(rs_h=0), dict(scale_x=2.0000001), dict(x2a=65),
                dict(x1a=30, x2a=26), dict(dx=1), dict(y2a=21)):
        with pytest.raises(lib.B2YError):
            mosaic(**bad)
    for bad in (dict(hsv=1, channels=1), dict(hsv=2), dict(flip=3), dict(slot=1), dict(im=[1e9, 0, 0, 0, 1, 0]),
                dict(im=[float("nan"), 0, 0, 0, 1, 0])):
        with pytest.raises(lib.B2YError):
            affine(**bad)
