"""Input pipeline on the device, inference slice (SURVEY section 8 f2): the reference's `letterbox`
(utils/datasets.py:611-646) and the BGR -> RGB / HWC -> CHW shuffle of its loaders (datasets.py:108-118, 180-186, 250-256)
as ONE kernel (csrc/preprocess.cu) that writes the uint8 NCHW tensor the model consumes (the stem kernel applies the
reference's `/ 256`).  Bit-exact against cv2.resize(INTER_LINEAR) + cv2.copyMakeBorder, which is what the reference calls.

    img, ratio, pad = letterbox(img0, new_shape=416)                # img0: HWC uint8 BGR (cv2.imread) on the device
    batch = letterbox_batch([img0, img1, ...], new_shape=640)       # [B, 3, 640, 640] uint8, auto=False
    pred = model(batch)                                             # uint8 in: "/ 256" happens inside the first conv

Host images (numpy arrays / CPU tensors) are copied to the device as they are (raw BGR bytes, the smallest form of the
image); resizing, padding, channel shuffle and the float conversion never touch the CPU.

DeviceEvalLoader replaces test.py's DataLoader over LoadImagesAndLabels(rect=True): load_image's INTER_AREA downscale,
the rect letterbox and the shuffle of a whole batch in one launch (b2y_load_batch_u8), bit-exact with the reference.

    results, maps = test.test(cfg, data, model=model, dataloader=DeviceEvalLoader(dataset, batch_size))

DeviceTrainLoader replaces train.py's DataLoader over LoadImagesAndLabels(augment=True): load_mosaic, random_affine,
augment_hsv, the flip and the shuffle of a whole batch in two launches (b2y_mosaic_u8, b2y_affine_hsv_u8), with the
reference's random draws, bit-exact with it.

    dataloader = DeviceTrainLoader(dataset, batch_size, shuffle=not opt.rect, sampler=None)
"""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import lib
from .lib import call, ptr, stream_ptr


def letterbox_params(shape, new_shape=(416, 416), auto=True, scaleFill=False, scaleup=True):
    """The host-side integer logic of datasets.py:614-640 for a source of `shape` = (height, width):
    returns (new_unpad (w, h), ratio, (dw, dh), (top, bottom, left, right))."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:                                  # only scale down (better test mAP)
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:                                         # minimum rectangle
        dw, dh = np.mod(dw, 64), np.mod(dh, 64)
    elif scaleFill:                                  # stretch (the reference passes (h, w) to cv2 here; kept)
        dw, dh = 0.0, 0.0
        new_unpad = new_shape
        ratio = new_shape[0] / shape[1], new_shape[1] / shape[0]
    dw /= 2
    dh /= 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return new_unpad, ratio, (dw, dh), (top, bottom, left, right)


DBL_EPSILON = 2.220446049250313e-16


def load_image_size(h0, w0, img_size):
    """The size load_image (datasets.py:511-531, augment=False) resizes a (h0, w0) source to: sources larger than
    img_size shrink with INTER_AREA to (int(h0 * r), int(w0 * r)), r = img_size / max(h0, w0); others stay as they are."""
    r = img_size / max(h0, w0)
    if r < 1:
        return int(h0 * r), int(w0 * r)
    return h0, w0


def inter_area_params(src_h, src_w, h, w):
    """cv2.resize's INTER_AREA set-up for a downscale (h, w <= src_h, src_w): returns (scale_x, scale_y, kx, ky).
    kx, ky > 0 are the integer factors of the block-mean path, which OpenCV takes when both scales are integers within
    DBL_EPSILON (saturate_cast<int>(double) rounds half to even, as Python's round does); 0, 0 = the fractional path."""
    scale_x = 1.0 / (w / src_w)
    scale_y = 1.0 / (h / src_h)
    kx, ky = round(scale_x), round(scale_y)
    if abs(scale_x - kx) < DBL_EPSILON and abs(scale_y - ky) < DBL_EPSILON:
        return scale_x, scale_y, kx, ky
    return scale_x, scale_y, 0, 0


def eval_labels(x, ratio, w, h, pad, out_h, out_w):
    """LoadImagesAndLabels.__getitem__'s label mapping (datasets.py:441-467) for one image without augmentation:
    normalised xywh (float32 [n, 5] with the class first) -> pixel xyxy through ratio and pad -> xywh normalised by the
    letterboxed (out_h, out_w).  The same numpy operations in the same order, with the scalar types the reference has:
    ratio and pad are numpy float64 (from its numpy batch shape), so under numpy 2's promotion each box coordinate is
    computed in float64 and rounded once into the float32 array; the divisions by the integer sizes stay float32."""
    if x.size == 0:
        return np.zeros((0, 5), np.float32)
    labels = x.copy()
    labels[:, 1] = ratio[0] * w * (x[:, 1] - x[:, 3] / 2) + pad[0]
    labels[:, 2] = ratio[1] * h * (x[:, 2] - x[:, 4] / 2) + pad[1]
    labels[:, 3] = ratio[0] * w * (x[:, 1] + x[:, 3] / 2) + pad[0]
    labels[:, 4] = ratio[1] * h * (x[:, 2] + x[:, 4] / 2) + pad[1]
    b = labels[:, 1:5]
    y = np.zeros_like(b)                             # utils.xyxy2xywh
    y[:, 0] = (b[:, 0] + b[:, 2]) / 2
    y[:, 1] = (b[:, 1] + b[:, 3]) / 2
    y[:, 2] = b[:, 2] - b[:, 0]
    y[:, 3] = b[:, 3] - b[:, 1]
    labels[:, 1:5] = y
    labels[:, [2, 4]] /= out_h
    labels[:, [1, 3]] /= out_w
    return labels


def _device_image(img0, device):
    if isinstance(img0, np.ndarray):
        img0 = torch.from_numpy(np.ascontiguousarray(img0))
    if img0.dim() == 2:
        img0 = img0[:, :, None]
    if img0.dtype != torch.uint8 or img0.dim() != 3:
        raise ValueError("letterbox expects an HWC uint8 image (cv2.imread layout)")
    if not img0.is_cuda:
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        img0 = img0.contiguous().to(device, non_blocking=True)
    return img0.contiguous()


def letterbox(img0, new_shape=(416, 416), color=(114, 114, 114), auto=True, scaleFill=False, scaleup=True,
              is_gray_scale=False, out=None, device=None, to_rgb=True):
    """Drop-in for datasets.letterbox + the loaders' `img[:, :, ::-1].transpose(2, 0, 1)`: returns
    (uint8 [C, H, W] device tensor in RGB order, ratio, (dw, dh)).  `out` = a preallocated [C, H, W] uint8 device view
    (e.g. one slot of a batch) to write into."""
    if not torch.cuda.is_available():
        raise lib.B2YError("letterbox runs on the CUDA device only (no CPU fallback)")
    c0 = color[0] if isinstance(color, (tuple, list)) else color
    if isinstance(color, (tuple, list)) and any(int(c) != int(c0) for c in color):
        raise NotImplementedError("letterbox border colour must be the same on all channels (the reference uses 114)")
    src = _device_image(img0, device if out is None else out.device)
    H, W, Cn = src.shape
    (rw, rh), ratio, pad, (top, bottom, left, right) = letterbox_params((H, W), new_shape, auto, scaleFill, scaleup)
    dh, dw = rh + top + bottom, rw + left + right
    if out is None:
        out = torch.empty((Cn, dh, dw), dtype=torch.uint8, device=src.device)
    if tuple(out.shape) != (Cn, dh, dw) or out.dtype != torch.uint8 or not out.is_contiguous():
        raise ValueError("letterbox: `out` must be a contiguous uint8 [%d, %d, %d] tensor" % (Cn, dh, dw))
    with torch.cuda.device(src.device):
        call("b2y_letterbox_u8", ptr(src), H, W, Cn, C.c_longlong(W * Cn), rh, rw, top, left, ptr(out), dh, dw,
             1 if (to_rgb and Cn == 3) else 0, int(c0), stream_ptr())
    return out, ratio, pad


def letterbox_batch(images, new_shape=640, scaleup=True, device=None):
    """Fixed-size batch (auto=False) of sources that are already `new_shape` or smaller, e.g. the output of load_image:
    list of HWC uint8 BGR images -> (uint8 [B, 3, H, W] RGB batch on the device, [ratio], [(dw, dh)]).  Larger sources
    are downscaled with letterbox's INTER_LINEAR, which is not what LoadImagesAndLabels does with raw cv2.imread images
    (load_image shrinks them with INTER_AREA first): build evaluation batches with DeviceEvalLoader."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    first = _device_image(images[0], device)
    batch = torch.empty((len(images), first.shape[2], new_shape[0], new_shape[1]), dtype=torch.uint8, device=first.device)
    ratios, pads = [], []
    for b, im in enumerate(images):
        _, r, p = letterbox(first if b == 0 else im, new_shape, auto=False, scaleup=scaleup, out=batch[b])
        ratios.append(r)
        pads.append(p)
    return batch, ratios, pads


class DeviceEvalLoader:
    """test.py's `DataLoader(dataset, batch_size, collate_fn=dataset.collate_fn)` over a LoadImagesAndLabels built with
    rect=True and no augmentation, with the images built on the device.  Iterating yields what that loader yields:
    (uint8 [B, C, H, W] device batch, float32 [nT, 6] device targets (image index, class, xywh normalised), paths,
    shapes = ((h0, w0), ((h / h0, w / w0), pad)) per image).

    `dataset` is the reference's dataset or any object with its attributes: img_files, labels, batch, batch_shapes,
    img_size, imgs (the --cache-images cache, with img_hw0 / img_hw), is_gray_scale, augment.  Sources are decoded with
    cv2.imread on host threads and copied to the device once, as raw bytes; INTER_AREA, border, channel shuffle and
    batching run in one launch per batch (b2y_load_batch_u8).  Labels are mapped on the host (a few floats per box, the
    reference's own numpy arithmetic) and reach the device in one copy per batch."""

    def __init__(self, dataset, batch_size, device=None, workers=None):
        if getattr(dataset, "augment", False):
            raise ValueError("DeviceEvalLoader builds evaluation batches only: the dataset has augment=True")
        if not getattr(dataset, "rect", True) or getattr(dataset, "batch_shapes", None) is None:
            raise ValueError("DeviceEvalLoader needs a rect=True dataset (rectangular batch shapes)")
        self.dataset = dataset
        self.batch_size = int(batch_size)
        self.device = None if device is None else torch.device(device)
        self.workers = workers or min(8, os.cpu_count() or 1)
        self._pool = None

    def __len__(self):
        return (len(self.dataset.img_files) + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        for b in range(len(self)):
            yield self.batch(b)

    def batch(self, b):
        """Batch b: (imgs, targets, paths, shapes)."""
        return self.device_batch(self.host_batch(b))

    def _read(self, index):
        ds = self.dataset
        imgs = getattr(ds, "imgs", None)
        if imgs is not None and imgs[index] is not None:        # --cache-images: load_image's output, kept in memory
            img = imgs[index]
            (h0, w0), hw = ds.img_hw0[index], ds.img_hw[index]
        else:
            import cv2
            path = ds.img_files[index]
            img = cv2.imread(path, flags=cv2.IMREAD_GRAYSCALE) if ds.is_gray_scale else cv2.imread(path)
            if img is None:
                raise FileNotFoundError("Image Not Found " + path)
            h0, w0 = img.shape[:2]
            hw = load_image_size(h0, w0, ds.img_size)
        img = np.ascontiguousarray(img)
        if img.ndim == 2:
            img = img[:, :, None]
        if img.dtype != np.uint8 or img.ndim != 3:
            raise ValueError("%s: expected an HWC uint8 image" % ds.img_files[index])
        return img, (h0, w0), tuple(hw)

    def host_batch(self, b):
        """Decode the sources of batch b (threads) and plan every item on the host: sizes, INTER_AREA path, border,
        labels, shapes.  Returns a list of per-image dicts."""
        ds = self.dataset
        idx = list(range(b * self.batch_size, min(len(ds.img_files), (b + 1) * self.batch_size)))
        if self._pool is None:
            self._pool = ThreadPoolExecutor(self.workers)
        reads = list(self._pool.map(self._read, idx)) if len(idx) > 1 else [self._read(i) for i in idx]
        plans = []
        for i, (img, (h0, w0), (h, w)) in zip(idx, reads):
            # the batch shape stays the numpy row it is in the reference: ratio and pad come out as numpy float64
            # scalars, which the label arithmetic below depends on
            shape = ds.batch_shapes[ds.batch[i]]
            (rw, rh), ratio, pad, (top, bottom, left, right) = letterbox_params((h, w), shape, auto=False, scaleup=False)
            if (rw, rh) != (w, h):
                raise NotImplementedError(
                    "%s: resized to %dx%d, it does not fit its batch shape %s; letterbox would resize it a second time"
                    % (ds.img_files[i], w, h, tuple(int(v) for v in shape)))
            src_h, src_w, cn = img.shape
            if cn != (1 if ds.is_gray_scale else 3):
                raise ValueError("%s: %d channels in a %s dataset" % (ds.img_files[i], cn,
                                                                     "gray-scale" if ds.is_gray_scale else "colour"))
            if (src_h, src_w) == (h, w):
                scales = (1.0, 1.0, 0, 0)
            elif h > src_h or w > src_w:
                raise NotImplementedError("%s: up-scaling (%dx%d -> %dx%d) is not part of evaluation loading"
                                          % (ds.img_files[i], src_w, src_h, w, h))
            else:
                scales = inter_area_params(src_h, src_w, h, w)
            out_h, out_w = h + top + bottom, w + left + right
            plans.append(dict(img=img, rs=(h, w), top=top, left=left, out=(out_h, out_w), scales=scales,
                              labels=eval_labels(ds.labels[i], ratio, w, h, pad, out_h, out_w),
                              path=ds.img_files[i], shapes=((h0, w0), ((h / h0, w / w0), pad))))
        if len({p["out"] for p in plans}) != 1:
            raise ValueError("batch %d mixes letterboxed shapes %s: the loader's batch_size must be the dataset's"
                             % (b, sorted({p["out"] for p in plans})))
        return plans

    def device_batch(self, plans):
        """One host-to-device copy of the sources and the item table, one launch for the images, one copy of the
        targets."""
        from .lib import LoadItem
        if not torch.cuda.is_available():
            raise lib.B2YError("DeviceEvalLoader runs on the CUDA device only (no CPU fallback)")
        if self.device is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        B, (H, W), cn = len(plans), plans[0]["out"], plans[0]["img"].shape[2]
        isz = C.sizeof(LoadItem)
        offs, total = [], isz * B
        for p in plans:
            total = (total + 15) // 16 * 16
            offs.append(total)
            total += p["img"].nbytes
        dev = torch.empty(total, dtype=torch.uint8, device=self.device)
        base = dev.data_ptr()
        items = (LoadItem * B)()
        host = np.empty(total, np.uint8)
        for k, (p, o) in enumerate(zip(plans, offs)):
            img = p["img"]
            sx, sy, kx, ky = p["scales"]
            items[k] = LoadItem(src=base + o, src_pitch=img.shape[1] * cn, src_h=img.shape[0], src_w=img.shape[1],
                                rs_h=p["rs"][0], rs_w=p["rs"][1], area_kx=kx, area_ky=ky, scale_x=sx, scale_y=sy,
                                top=p["top"], left=p["left"], slot=k)
            host[o:o + img.nbytes] = img.reshape(-1)
        host[:isz * B] = np.frombuffer(bytes(items), np.uint8)
        dev.copy_(torch.from_numpy(host))
        out = torch.empty((B, cn, H, W), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            call("b2y_load_batch_u8", C.cast(items, C.c_void_p), ptr(dev), B, ptr(out), B, cn, H, W,
                 1 if cn == 3 else 0, 114, stream_ptr())
        labels = []
        for k, p in enumerate(plans):
            lo = torch.zeros((len(p["labels"]), 6))
            if len(p["labels"]):
                lo[:, 1:] = torch.from_numpy(p["labels"])
            lo[:, 0] = k
            labels.append(lo)
        targets = torch.cat(labels, 0).to(self.device)
        return out, targets, tuple(p["path"] for p in plans), tuple(p["shapes"] for p in plans)


def train_tile_size(h0, w0, img_size):
    """The size load_image (datasets.py:511-531) gives a (h0, w0) source with augment=True: any r = img_size /
    max(h0, w0) != 1 resizes with INTER_LINEAR, up or down, to (int(h0 * r), int(w0 * r))."""
    r = img_size / max(h0, w0)
    if r != 1:
        return int(h0 * r), int(w0 * r)
    return h0, w0


def mosaic_rects(k, xc, yc, w, h, s):
    """load_mosaic's placement of tile k (datasets.py:565-579), its x2b = max(xc, w) of tile 2 included, with numpy's
    slice clamping applied to the tile side: ((x1a, y1a, x2a, y2a), (x1b, y1b, x2b, y2b))."""
    if k == 0:
        x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
        x1b, y1b, x2b, y2b = w - (x2a - x1a), h - (y2a - y1a), w, h
    elif k == 1:
        x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
        x1b, y1b, x2b, y2b = 0, h - (y2a - y1a), min(w, x2a - x1a), h
    elif k == 2:
        x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
        x1b, y1b, x2b, y2b = w - (x2a - x1a), 0, max(xc, w), min(y2a - y1a, h)
    else:
        x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
        x1b, y1b, x2b, y2b = 0, 0, min(w, x2a - x1a), min(y2a - y1a, h)
    x1b, x2b, _ = slice(x1b, x2b).indices(w)
    y1b, y2b, _ = slice(y1b, y2b).indices(h)
    return (x1a, y1a, x2a, y2a), (x1b, y1b, x2b, y2b)


def _xyxy2xywh(b):
    y = np.zeros_like(b)
    y[:, 0] = (b[:, 0] + b[:, 2]) / 2
    y[:, 1] = (b[:, 1] + b[:, 3]) / 2
    y[:, 2] = b[:, 2] - b[:, 0]
    y[:, 3] = b[:, 3] - b[:, 1]
    return y


def train_labels(tiles, s, M, scale, flip):
    """Labels of one mosaic item, restating the reference's numpy arithmetic and dtypes: load_mosaic's pixel xyxy per
    tile (float32 labels, Python-int sizes and pads) and clip to [0, 2s]; random_affine's float64 `xy @ M.T`, clip,
    filter (w > 4, h > 4, area ratio > 0.2, aspect < 10) and cast back; xyxy2xywh, the normalisation by s and the
    left-right flip.  tiles: [(labels float32 [n, 5], w, h, padw, padh)]."""
    labels4 = []
    for x, w, h, padw, padh in tiles:
        labels = x.copy()
        if x.size > 0:
            labels[:, 1] = w * (x[:, 1] - x[:, 3] / 2) + padw
            labels[:, 2] = h * (x[:, 2] - x[:, 4] / 2) + padh
            labels[:, 3] = w * (x[:, 1] + x[:, 3] / 2) + padw
            labels[:, 4] = h * (x[:, 2] + x[:, 4] / 2) + padh
        labels4.append(labels)
    targets = np.concatenate(labels4, 0)
    np.clip(targets[:, 1:], 0, 2 * s, out=targets[:, 1:])
    n = len(targets)
    if n:
        width = height = s
        xy = np.ones((n * 4, 3))
        xy[:, :2] = targets[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(n * 4, 2)
        xy = (xy @ M.T)[:, :2].reshape(n, 8)
        x = xy[:, [0, 2, 4, 6]]
        y = xy[:, [1, 3, 5, 7]]
        xy = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
        xy[:, [0, 2]] = xy[:, [0, 2]].clip(0, width)
        xy[:, [1, 3]] = xy[:, [1, 3]].clip(0, height)
        w = xy[:, 2] - xy[:, 0]
        h = xy[:, 3] - xy[:, 1]
        area = w * h
        area0 = (targets[:, 3] - targets[:, 1]) * (targets[:, 4] - targets[:, 2])
        ar = np.maximum(w / (h + 1e-16), h / (w + 1e-16))
        i = (w > 4) & (h > 4) & (area / (area0 * scale + 1e-16) > 0.2) & (ar < 10)
        targets = targets[i]
        targets[:, 1:5] = xy[i]
    if len(targets):
        targets[:, 1:5] = _xyxy2xywh(targets[:, 1:5])
        targets[:, [2, 4]] /= s
        targets[:, [1, 3]] /= s
        if flip:
            targets[:, 1] = 1 - targets[:, 1]
    return targets


def hsv_luts(r):
    """augment_hsv's three uint8 LUTs (datasets.py:534-545) for the gains r (float64 [3]), as one [768] array."""
    x = np.arange(0, 256, dtype=np.int16)
    lut_hue = ((x * r[0]) % 180).astype(np.uint8)
    lut_sat = np.clip(x * r[1], 0, 255).astype(np.uint8)
    lut_val = np.clip(x * r[2], 0, 255).astype(np.uint8)
    return np.concatenate((lut_hue, lut_sat, lut_val))


class DeviceTrainLoader:
    """train.py's `DataLoader(dataset, batch_size, shuffle, sampler, collate_fn=dataset.collate_fn)` over a
    LoadImagesAndLabels built with augment=True and rect=False (mosaic training), with the images built on the device.
    Iterating yields what that loader yields: (uint8 [B, C, s, s] device batch, float32 [nT, 6] device targets (image
    index, class, xywh normalised), paths, shapes = (None,) * B).

    The index order is a DataLoader's over the same sampler (RandomSampler when shuffle, the given `sampler`, e.g. a
    DistributedSampler, whose set_epoch works through `.sampler`), and the `random` / `np.random` draws of every item
    are made in the order a num_workers=0 DataLoader makes them, before any pixel is touched: the mosaic centre and
    the 3 extra indices, random_affine's six draws, augment_hsv's gains (colour only), the flip.  Each distinct image
    of a batch is taken once, from the --cache-images arrays (imgs, img_hw0, img_hw) when the dataset has them, else
    by cv2.imread on host threads; sources and both item tables reach the device in one copy.  b2y_mosaic_u8 builds the
    2s x 2s canvases (load_image's INTER_LINEAR for uncached sources) in a workspace kept across batches;
    b2y_affine_hsv_u8 warps, applies the HSV LUTs, flips and reverses the channels into the batch.  Labels are mapped
    on the host with the reference's numpy arithmetic (train_labels) and copied once per batch.

    `dataset` is the reference's dataset or any object with its attributes: img_files, labels, img_size, hyp, augment,
    rect, image_weights (with indices), is_gray_scale, imgs (+ img_hw0, img_hw)."""

    def __init__(self, dataset, batch_size, shuffle=True, sampler=None, drop_last=False, device=None, workers=None):
        if not getattr(dataset, "augment", False):
            raise ValueError("DeviceTrainLoader builds augmented training batches: the dataset has augment=False "
                             "(build evaluation batches with DeviceEvalLoader)")
        if getattr(dataset, "rect", False):
            raise ValueError("DeviceTrainLoader builds mosaic batches: rect=True training (letterbox after load_image) "
                             "is not supported")
        self.dataset = dataset
        self.batch_size = int(batch_size)
        self._index = torch.utils.data.DataLoader(range(len(dataset.img_files)), batch_size=self.batch_size,
                                                  shuffle=shuffle, sampler=sampler, drop_last=drop_last,
                                                  collate_fn=list)
        self.sampler = self._index.sampler
        self.device = None if device is None else torch.device(device)
        self.workers = workers or min(8, os.cpu_count() or 1)
        self._pool = None
        self._canvas = None

    def __len__(self):
        return len(self._index)

    def __iter__(self):
        for indices in self._index:
            yield self.device_batch(self.host_batch(indices))

    def _read(self, index):
        ds = self.dataset
        imgs = getattr(ds, "imgs", None)
        if imgs is not None and imgs[index] is not None:         # --cache-images: load_image's output
            img, hw = imgs[index], tuple(ds.img_hw[index])
        else:
            import cv2
            path = ds.img_files[index]
            img = cv2.imread(path, flags=cv2.IMREAD_GRAYSCALE) if ds.is_gray_scale else cv2.imread(path)
            if img is None:
                raise FileNotFoundError("Image Not Found " + path)
            hw = train_tile_size(img.shape[0], img.shape[1], ds.img_size)
        img = np.ascontiguousarray(img)
        if img.ndim == 2:
            img = img[:, :, None]
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != (1 if ds.is_gray_scale else 3):
            raise ValueError("%s: expected an HWC uint8 %s image" % (ds.img_files[index],
                                                                    "gray-scale" if ds.is_gray_scale else "colour"))
        return img, hw

    def draws(self, indices):
        """The random draws of the items of one batch, in __getitem__'s order: per item (index, xc, yc, the 4 tile
        indices, (angle, scale, tx, ty, shear x, shear y), HSV gains or None, flip)."""
        import random
        ds = self.dataset
        s, hyp = ds.img_size, ds.hyp
        out = []
        for index in indices:
            if getattr(ds, "image_weights", False):
                index = ds.indices[index]
            xc, yc = [int(random.uniform(s * 0.5, s * 1.5)) for _ in range(2)]
            tiles = [index] + [random.randint(0, len(ds.labels) - 1) for _ in range(3)]
            a = random.uniform(-hyp["degrees"], hyp["degrees"])
            sc = random.uniform(1 - hyp["scale"], 1 + hyp["scale"])
            tx = random.uniform(-hyp["translate"], hyp["translate"])
            ty = random.uniform(-hyp["translate"], hyp["translate"])
            shx = random.uniform(-hyp["shear"], hyp["shear"])
            shy = random.uniform(-hyp["shear"], hyp["shear"])
            gains = None
            if not ds.is_gray_scale:
                gains = np.random.uniform(-1, 1, 3) * [hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]] + 1
            flip = random.random() < 0.5
            out.append((index, xc, yc, tiles, (a, sc, tx, ty, shx, shy), gains, flip))
        return out

    def host_batch(self, indices):
        """Draw, decode (threads) and plan the items of one batch on the host: tiles and their rectangles, the affine
        map and its inverse, LUTs, flips, labels.  Returns (sources {index: (img, (h, w))}, [per-item dict])."""
        import math
        import cv2
        ds = self.dataset
        s = ds.img_size
        draws = self.draws(indices)
        need = sorted({i for d in draws for i in d[3]})
        if self._pool is None:
            self._pool = ThreadPoolExecutor(self.workers)
        reads = list(self._pool.map(self._read, need)) if len(need) > 1 else [self._read(i) for i in need]
        sources = dict(zip(need, reads))
        plans = []
        for index, xc, yc, tiles, (a, sc, tx, ty, shx, shy), gains, flip in draws:
            rects, tile_labels = [], []
            for k, i in enumerate(tiles):
                h, w = sources[i][1]
                (x1a, y1a, x2a, y2a), (x1b, y1b, x2b, y2b) = mosaic_rects(k, xc, yc, w, h, s)
                if (x2a - x1a, y2a - y1a) != (max(x2b - x1b, 0), max(y2b - y1b, 0)):
                    raise ValueError("%s: mosaic tile %d does not fit its rectangle" % (ds.img_files[i], k))
                rects.append(((x1a, y1a, x2a, y2a), (x1b - x1a, y1b - y1a)))
                tile_labels.append((ds.labels[i], w, h, x1a - x1b, y1a - y1b))
            # random_affine(border=-s // 2) on the 2s x 2s canvas: M = S @ T @ R, as the reference composes it
            border = -s // 2
            R = np.eye(3)
            R[:2] = cv2.getRotationMatrix2D(angle=a, center=(2 * s / 2, 2 * s / 2), scale=sc)
            T = np.eye(3)
            T[0, 2] = tx * (2 * s) + border
            T[1, 2] = ty * (2 * s) + border
            S = np.eye(3)
            S[0, 1] = math.tan(shx * math.pi / 180)
            S[1, 0] = math.tan(shy * math.pi / 180)
            M = S @ T @ R
            im = cv2.invertAffineTransform(M[:2])
            plans.append(dict(index=index, tiles=tiles, rects=rects, M=M, im=im, flip=flip,
                              lut=None if gains is None else hsv_luts(gains),
                              labels=train_labels(tile_labels, s, M, sc, flip), path=ds.img_files[index]))
        return sources, plans

    def device_batch(self, planned):
        """One host-to-device copy of the sources and both item tables, b2y_mosaic_u8 then b2y_affine_hsv_u8, one
        copy of the targets."""
        from .lib import AffineItem, MosaicItem
        if not torch.cuda.is_available():
            raise lib.B2YError("DeviceTrainLoader runs on the CUDA device only (no CPU fallback)")
        if self.device is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        sources, plans = planned
        s, B = self.dataset.img_size, len(plans)
        cn = next(iter(sources.values()))[0].shape[2]
        off_aff = C.sizeof(MosaicItem) * B
        total = off_aff + C.sizeof(AffineItem) * B
        offs = {}
        for i, (img, _) in sources.items():
            total = (total + 15) // 16 * 16
            offs[i] = total
            total += img.nbytes
        dev = torch.empty(total, dtype=torch.uint8, device=self.device)
        base = dev.data_ptr()
        host = np.empty(total, np.uint8)
        for i, (img, _) in sources.items():
            host[offs[i]:offs[i] + img.nbytes] = img.reshape(-1)
        mos, aff = (MosaicItem * B)(), (AffineItem * B)()
        for k, p in enumerate(plans):
            mos[k].slot = aff[k].slot = k
            for t, (i, ((x1a, y1a, x2a, y2a), (dx, dy))) in enumerate(zip(p["tiles"], p["rects"])):
                img, (h, w) = sources[i]
                sh, sw = img.shape[:2]
                mos[k].tiles[t] = lib.MosaicTile(src=base + offs[i], src_pitch=sw * cn, src_h=sh, src_w=sw, rs_h=h,
                                                 rs_w=w, scale_x=1.0 / (w / sw), scale_y=1.0 / (h / sh), x1a=x1a,
                                                 y1a=y1a, x2a=x2a, y2a=y2a, dx=dx, dy=dy)
            aff[k].im[:] = [float(v) for v in p["im"].reshape(-1)]
            if p["lut"] is not None:
                C.memmove(aff[k].lut, p["lut"].ctypes.data, 768)
                aff[k].hsv = 1
            aff[k].flip = 1 if p["flip"] else 0
        host[:off_aff] = np.frombuffer(bytes(mos), np.uint8)
        host[off_aff:off_aff + C.sizeof(AffineItem) * B] = np.frombuffer(bytes(aff), np.uint8)
        dev.copy_(torch.from_numpy(host))
        if self._canvas is None or self._canvas.shape[0] < B or tuple(self._canvas.shape[1:]) != (2 * s, 2 * s, cn):
            self._canvas = torch.empty((max(B, self.batch_size), 2 * s, 2 * s, cn), dtype=torch.uint8,
                                       device=self.device)
        out = torch.empty((B, cn, s, s), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            call("b2y_mosaic_u8", C.cast(mos, C.c_void_p), ptr(dev), B, ptr(self._canvas), self._canvas.shape[0], cn,
                 s, stream_ptr())
            call("b2y_affine_hsv_u8", C.cast(aff, C.c_void_p), C.c_void_p(base + off_aff), B, ptr(self._canvas),
                 ptr(out), B, cn, s, stream_ptr())
        labels = []
        for k, p in enumerate(plans):
            lo = torch.zeros((len(p["labels"]), 6))
            if len(p["labels"]):
                lo[:, 1:] = torch.from_numpy(p["labels"])
            lo[:, 0] = k
            labels.append(lo)
        targets = torch.cat(labels, 0).to(self.device)
        return out, targets, tuple(p["path"] for p in plans), (None,) * B
