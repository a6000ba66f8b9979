"""GPU parity tests of the individual CUDA kernels (called through the C ABI via b200yolo.ops).

Reference for each kernel is plain PyTorch fp32 on the *same fp16-rounded operands* (SURVEY.md section 7:
gate convs on max|d| <= tol * rms(y), not on elementwise-relative error).
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from b200yolo import ops
    return ops


def _ref_act(y, act, slope=0.1):
    if act == "leaky":
        return F.leaky_relu(y, slope)
    if act == "mish":
        return y * torch.tanh(F.softplus(y))
    if act == "relu":
        return F.relu(y)
    if act == "relu6":
        return F.relu6(y)
    if act == "h_swish":
        return y * (F.relu6(y + 3.0) / 6.0)
    if act == "swish":
        return y * torch.sigmoid(y)
    return y


def conv_case(B, H, W, Cin, Cout, k, stride, act="leaky", residual=False, out_f32=False, in_extra=0, out_extra=0,
              seed=0):
    """Returns (max abs err, rms of reference)."""
    ops = _ops()
    g = torch.Generator(device="cpu").manual_seed(seed)
    pad = (k - 1) // 2
    x = (torch.randn(B, Cin, H, W, generator=g) * 1.0).half().float()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k)).half().float()
    bias = torch.randn(Cout, generator=g) * 0.5
    ref = F.conv2d(x.double(), w.double(), bias.double(), stride=stride, padding=pad).float()
    ref = _ref_act(ref, act)
    Ho, Wo = ref.shape[2], ref.shape[3]
    res = None
    if residual:
        res = (torch.randn(B, Cout, Ho, Wo, generator=g)).half().float()
        ref = ref + res
    dev = "cuda"
    # NHWC fp16 input living inside a wider buffer (exercise pitch / channel-offset views)
    xbuf = torch.zeros(B, H, W, Cin + in_extra, dtype=torch.float16, device=dev)
    xv = xbuf[..., in_extra:] if in_extra else xbuf
    xv.copy_(x.permute(0, 2, 3, 1).half())
    wp = w.permute(0, 2, 3, 1).contiguous().half().to(dev)
    obuf = torch.zeros(B, Ho, Wo, Cout + out_extra, dtype=torch.float32 if out_f32 else torch.float16, device=dev)
    ov = obuf[..., out_extra:] if out_extra else obuf
    rv = res.permute(0, 2, 3, 1).contiguous().half().to(dev) if residual else None
    ops.conv2d(xv, wp, bias.to(dev), k, stride, pad, act=act, residual=rv, out=ov)
    torch.cuda.synchronize()
    got = ov.float().permute(0, 3, 1, 2).cpu()
    if out_extra:
        assert float(obuf[..., :out_extra].abs().max()) == 0.0, "wrote outside the channel slice"
    err = (got - ref).abs().max().item()
    rms = ref.pow(2).mean().sqrt().item()
    return err, rms


CONV_CASES = [
    # (B, H, W, Cin, Cout, k, stride, act, residual, out_f32, in_extra, out_extra)
    (1, 16, 16, 64, 64, 1, 1, "linear", False, False, 0, 0),      # plain GEMM, 2-D tiled TMA
    (2, 20, 20, 128, 256, 1, 1, "leaky", False, False, 0, 0),
    (2, 20, 20, 64, 128, 3, 1, "leaky", False, False, 0, 0),      # im2col TMA, swizzle 128
    (2, 20, 20, 128, 256, 3, 1, "leaky", True, False, 0, 0),      # + residual
    (1, 40, 40, 32, 64, 3, 1, "leaky", False, False, 0, 0),       # Cin=32 -> 64B swizzle
    (1, 40, 40, 16, 32, 3, 1, "leaky", False, False, 0, 0),       # Cin=16 -> 32B swizzle
    (2, 40, 40, 64, 128, 3, 2, "leaky", False, False, 0, 0),      # stride 2
    (1, 38, 26, 64, 64, 3, 2, "mish", False, False, 0, 0),        # non-square, ragged M tile
    (2, 13, 13, 256, 512, 3, 1, "mish", False, False, 0, 0),      # 2 N tiles
    (3, 10, 10, 512, 255, 1, 1, "linear", False, True, 0, 0),     # yolo head: N=255, fp32 out
    (2, 20, 20, 384, 128, 1, 1, "leaky", False, False, 0, 0),     # K=384 (route concat input)
    (2, 20, 20, 128, 64, 1, 1, "leaky", False, False, 64, 0),     # input is a channel slice of a wider buffer
    (2, 20, 20, 64, 128, 3, 1, "leaky", False, False, 0, 128),    # output into a concat slot
    (1, 52, 52, 128, 256, 3, 1, "relu6", False, False, 0, 0),
    (1, 24, 24, 96, 48, 1, 1, "h_swish", False, False, 0, 0),     # K=96 -> 64B swizzle, Cout=48
]


@pytest.mark.parametrize("case", CONV_CASES, ids=[str(c) for c in CONV_CASES])
def test_conv2d_tc(case):
    err, rms = conv_case(*case)
    out_f32 = case[9]
    tol = (2e-5 if out_f32 else 2e-3) * max(rms, 1.0)  # fp16 store: 2^-11 relative of |y| ~ a few rms
    assert err <= tol + (0 if out_f32 else 4e-3 * rms), "max err %g rms %g" % (err, rms)


def test_conv2d_large_multiwave():
    # more tiles than SMs -> exercises the persistent loop, the smem ring wrap and the accumulator staging reuse
    err, rms = conv_case(4, 80, 80, 128, 256, 3, 1, "leaky")
    assert err <= 6e-3 * max(rms, 1.0)


def test_conv_stats():
    ops = _ops()
    g = torch.Generator().manual_seed(3)
    B, H, W, Cin, Cout = 2, 20, 20, 64, 128
    x = torch.randn(B, Cin, H, W, generator=g).half().float()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / 24).half().float()
    ref = F.conv2d(x.double(), w.double(), None, padding=1)
    s1 = ref.sum(dim=(0, 2, 3)).float()
    s2 = (ref * ref).sum(dim=(0, 2, 3)).float()
    xv = x.permute(0, 2, 3, 1).contiguous().half().cuda()
    wp = w.permute(0, 2, 3, 1).contiguous().half().cuda()
    st = (torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda"))
    y = ops.conv2d(xv, wp, None, 3, 1, 1, stats=st)
    torch.cuda.synchronize()
    assert (y.float().permute(0, 3, 1, 2).cpu() - ref.float()).abs().max() < 5e-3
    assert torch.allclose(st[0].cpu(), s1, rtol=1e-4, atol=1e-2)
    assert torch.allclose(st[1].cpu(), s2, rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("shape", [(2, 40, 36, 64), (3, 22, 50, 128), (1, 96, 64, 64)], ids=str)
def test_conv_s2_pixel_pair_layout(shape):
    """B2Y_WLAYOUT_S2_PAIRS (include/b200yolo.h): the 3x3 / stride-2 / Cin = 32 layer through the pixel-pair view (3 x 2
    window, stride 2 x 1) against fp64 and against the dense-layout launch of the same kernel; with statistics and with
    a residual; rejected for odd widths / non-dense inputs."""
    from b200yolo.lib import B2YError, WLAYOUT_S2_PAIRS
    ops = _ops()
    B, H, W, Cout = shape
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, 32, H, W, generator=g).half().float()
    w = (torch.randn(Cout, 32, 3, 3, generator=g) / 17).half().float()
    b = torch.randn(Cout, generator=g)
    ref = F.leaky_relu(F.conv2d(x.double(), w.double(), b.double(), stride=2, padding=1), 0.1).float()
    xv = x.permute(0, 2, 3, 1).contiguous().half().cuda()
    wd = w.permute(0, 2, 3, 1).contiguous().half().cuda()
    wp = ops.s2_pair_weights(w.cuda()).half()
    res = torch.randn(ref.shape, generator=g).half()
    resv = res.permute(0, 2, 3, 1).contiguous().cuda()
    y_pair = ops.conv2d(xv, wp, b.cuda(), 3, 2, 1, act="leaky", residual=resv, w_layout=WLAYOUT_S2_PAIRS)
    y_dense = ops.conv2d(xv, wd, b.cuda(), 3, 2, 1, act="leaky", residual=resv)
    torch.cuda.synchronize()
    got = y_pair.float().permute(0, 3, 1, 2).cpu()
    want = ref + res.float()
    assert (got - want).abs().max() <= 4e-3 * max(1.0, want.abs().max().item())
    # same products, different summation order inside the tensor core: at most an fp16 ulp apart
    assert (y_pair.float() - y_dense.float()).abs().max() <= 2.0 ** -9 * max(1.0, want.abs().max().item())
    st = (torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda"))
    ops.conv2d(xv, wp, None, 3, 2, 1, stats=st, w_layout=WLAYOUT_S2_PAIRS)
    raw = F.conv2d(x.double(), w.double(), None, stride=2, padding=1)
    assert torch.allclose(st[0].cpu(), raw.sum(dim=(0, 2, 3)).float(), rtol=1e-4, atol=1e-2)
    assert torch.allclose(st[1].cpu(), (raw * raw).sum(dim=(0, 2, 3)).float(), rtol=1e-4, atol=1e-2)
    with pytest.raises(B2YError):
        ops.conv2d(xv[:, :, :W - 1].contiguous(), wp, None, 3, 2, 1, w_layout=WLAYOUT_S2_PAIRS)      # odd width
    wide = torch.zeros(B, H, W, 64, dtype=torch.float16, device="cuda")
    with pytest.raises(B2YError):
        ops.conv2d(wide[..., :32], wp, None, 3, 2, 1, w_layout=WLAYOUT_S2_PAIRS)                     # pitch != in_c


def test_stem_conv():
    ops = _ops()
    g = torch.Generator().manual_seed(1)
    x = torch.rand(2, 3, 64, 48, generator=g)
    w = torch.randn(32, 3, 3, 3, generator=g) / 5
    b = torch.randn(32, generator=g)
    for stride in (1, 2):
        ref = F.leaky_relu(F.conv2d(x, w, b, stride=stride, padding=1), 0.1)
        y = ops.stem_conv(x.cuda(), w.cuda(), b.cuda(), 3, stride, 1, act="leaky")
        torch.cuda.synchronize()
        got = y.float().permute(0, 3, 1, 2).cpu()
        assert (got - ref).abs().max() <= 2e-3 * max(1.0, ref.abs().max().item())
    # Cout = 16 (yolov3-tiny stem)
    w16 = torch.randn(16, 3, 3, 3, generator=g) / 5
    ref = F.leaky_relu(F.conv2d(x, w16, None, stride=1, padding=1), 0.1)
    y = ops.stem_conv(x.cuda(), w16.cuda(), None, 3, 1, 1, act="leaky")
    assert (y.float().permute(0, 3, 1, 2).cpu() - ref).abs().max() <= 2e-3 * max(1.0, ref.abs().max().item())
    # the first layers that no im2col kernel is compiled for (layout.stem_path): 5x5 and 7x7, 4 channels at 3x3, and
    # 1, 2 and 4 input channels
    for cin, k, stride, cout in ((3, 5, 1, 32), (1, 7, 1, 32), (2, 5, 2, 64), (4, 3, 1, 32), (4, 7, 2, 16),
                                 (2, 7, 1, 24), (1, 5, 2, 32)):
        xk = torch.rand(2, cin, 40, 56, generator=g)
        wk = torch.randn(cout, cin, k, k, generator=g) / (cin * k)
        bk = torch.randn(cout, generator=g)
        ref = F.leaky_relu(F.conv2d(xk, wk, bk, stride=stride, padding=k // 2), 0.1)
        y = ops.stem_conv(xk.cuda(), wk.cuda(), bk.cuda(), k, stride, k // 2, act="leaky")
        got = y.float().permute(0, 3, 1, 2).cpu()
        assert got.shape == ref.shape
        assert (got - ref).abs().max() <= 2e-3 * max(1.0, ref.abs().max().item()), (cin, k, stride, cout)


@pytest.mark.parametrize("cin,k,stride,cout", [(3, 3, 1, 32), (3, 3, 2, 32), (3, 3, 1, 16), (1, 5, 1, 32), (2, 3, 1, 32),
                                             (4, 1, 2, 72)])
def test_stem_conv_tensor_core(cin, k, stride, cout):
    """im2col workspace + GEMM stem: one 32-column im2col row per output pixel (B2Y_STEM_IM2COL_SHAPES)."""
    ops = _ops()
    g = torch.Generator().manual_seed(11)
    x = torch.rand(2, cin, 40, 56, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k)
    b = torch.randn(cout, generator=g)
    ref = F.leaky_relu(F.conv2d(x.half().float(), w.half().float(), b, stride=stride, padding=k // 2), 0.1)
    ws = ops.pack_stem_weights(w.cuda())
    y, _ = ops.stem_conv_tc(x.cuda(), ws, b.cuda(), cin, k, stride, k // 2, act="leaky")
    torch.cuda.synchronize()
    got = y.float().permute(0, 3, 1, 2).cpu()
    assert got.shape == ref.shape
    assert (got - ref).abs().max() <= 2e-3 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("cin,k,stride,cout,dtype", [
    (3, 3, 1, 32, "f32"), (3, 3, 2, 32, "f16"), (3, 3, 1, 16, "u8"), (1, 5, 1, 32, "f32"), (3, 3, 1, 64, "u8256"),
    (3, 3, 1, 48, "f32"), (2, 3, 1, 32, "f32"), (4, 1, 2, 64, "f16")])
def test_stem_conv_fused(cin, k, stride, cout, dtype):
    """Fused stem: the CTA builds the im2col tile in smem from the NCHW image (fp32 / fp16 / uint8 with /255)."""
    ops = _ops()
    g = torch.Generator().manual_seed(12)
    B, H, W = 3, 44, 72            # 3*44*72 = 9504 pixels: 74.25 tiles -> partial last tile, several tiles per CTA group
    if dtype in ("u8", "u8256"):
        x = torch.randint(0, 256, (B, cin, H, W), generator=g, dtype=torch.uint8)
        div = 255.0 if dtype == "u8" else 256.0
        xf = x.float() / div
    elif dtype == "f16":
        x = torch.rand(B, cin, H, W, generator=g).half()
        xf, div = x.float(), 1.0
    else:
        x = torch.rand(B, cin, H, W, generator=g)
        xf, div = x, 1.0
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k)
    b = torch.randn(cout, generator=g)
    for act, fn in (("leaky", lambda t: F.leaky_relu(t, 0.1)), ("mish", lambda t: t * torch.tanh(F.softplus(t)))):
        ref = fn(F.conv2d(xf.half().float(), w.half().float(), b, stride=stride, padding=k // 2))
        ws = ops.pack_stem_weights(w.cuda())
        assert ws.dim() == 2
        y = ops.stem_conv_fused(x.cuda(), ws, b.cuda(), k, stride, k // 2, act=act, x_div=div)
        torch.cuda.synchronize()
        got = y.float().permute(0, 3, 1, 2).cpu()
        assert got.shape == ref.shape
        assert (got - ref).abs().max() <= 2e-3 * max(1.0, ref.abs().max().item()), (act, (got - ref).abs().max())


@pytest.mark.parametrize("cin,cout,k,stride,res", [(32, 64, 3, 1, True), (32, 64, 3, 2, False), (64, 32, 1, 1, False),
                                                  (128, 64, 1, 1, False)])
def test_conv_weight_stationary_many_tiles(cin, cout, k, stride, res):
    """More M tiles than SMs and a weight panel that fits in smem: the weight-stationary launch (whole panel loaded once
    per CTA, the ring carries A only), 8 epilogue warps on alternate tiles, TMA-store epilogue with a partial last tile."""
    ops = _ops()
    g = torch.Generator().manual_seed(21)
    B, H, W = 2, 110, 100                       # 22000 pixels = 171.9 tiles > 132 SMs
    x = torch.randn(B, H, W, cin, generator=g).half()
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).half()
    b = torch.randn(cout, generator=g)
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    r = torch.randn(B, Ho, Wo, cout, generator=g).half() if res else None
    ref = F.leaky_relu(F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, stride=stride, padding=k // 2), 0.1)
    if res:
        ref = ref + r.float().permute(0, 3, 1, 2)
    wp = w.permute(0, 2, 3, 1).contiguous().cuda()
    y = ops.conv2d(x.cuda(), wp, b.cuda(), k, stride, k // 2, act="leaky", residual=r.cuda() if res else None)
    torch.cuda.synchronize()
    got = y.float().permute(0, 3, 1, 2).cpu()
    assert got.shape == ref.shape
    assert (got - ref).abs().max() <= 4e-3 * max(1.0, ref.abs().max().item())


def test_pack_weights_bn_fold():
    ops = _ops()
    g = torch.Generator().manual_seed(2)
    O, I, k = 64, 32, 3
    w = torch.randn(O, I, k, k, generator=g)
    gamma, beta = torch.rand(O, generator=g) + 0.5, torch.randn(O, generator=g)
    mean, var = torch.randn(O, generator=g) * 0.1, torch.rand(O, generator=g) + 0.5
    eps = 1e-5
    wp, bias, w32 = ops.pack_conv_weights(w.cuda(), None, (gamma.cuda(), beta.cuda(), mean.cuda(), var.cuda()), eps,
                                          want_fp32=True)
    scale = gamma / torch.sqrt(eps + var)
    wref = w * scale.view(-1, 1, 1, 1)
    bref = beta - gamma * mean / torch.sqrt(var + eps)
    assert torch.allclose(w32.cpu(), wref, rtol=1e-6, atol=1e-7)
    assert torch.allclose(bias.cpu(), bref, rtol=1e-6, atol=1e-6)
    assert torch.equal(wp.cpu(), wref.permute(0, 2, 3, 1).contiguous().half()) or \
        (wp.cpu().float() - wref.permute(0, 2, 3, 1)).abs().max() < 1e-3


def test_pointwise_layers():
    ops = _ops()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 64, 13, 13, generator=g).half()
    xn = x.permute(0, 2, 3, 1).contiguous().cuda()
    # upsample
    up = ops.upsample(xn, 2)
    assert torch.equal(up.permute(0, 3, 1, 2).cpu(), F.interpolate(x.float(), scale_factor=2).half())
    # maxpool SPP kernels, stride 1
    for k in (5, 9, 13):
        mp = ops.maxpool(xn, k, 1)
        assert torch.equal(mp.permute(0, 3, 1, 2).cpu(), F.max_pool2d(x.float(), k, 1, (k - 1) // 2).half())
    mp = ops.maxpool(xn[:, :12, :12].contiguous(), 2, 2)
    assert torch.equal(mp.permute(0, 3, 1, 2).cpu(), F.max_pool2d(x[:, :, :12, :12].float(), 2, 2).half())
    # yolov3-tiny ZeroPad2d((0,1,0,1)) + MaxPool2d(2,1)
    mp = ops.maxpool(xn, 2, 1, tiny_pad=True)
    ref = F.max_pool2d(F.pad(x.float(), (0, 1, 0, 1)), 2, 1).half()
    assert torch.equal(mp.permute(0, 3, 1, 2).cpu(), ref)
    # add / copy into a slice
    y = torch.randn(2, 64, 13, 13, generator=g).half()
    yn = y.permute(0, 2, 3, 1).contiguous().cuda()
    s = ops.add(xn, yn)
    assert torch.equal(s.permute(0, 3, 1, 2).cpu(), (x.float() + y.float()).half())
    buf = torch.zeros(2, 13, 13, 192, dtype=torch.float16, device="cuda")
    ops.copy_channels(xn, buf[..., 64:128])
    assert torch.equal(buf[..., 64:128].cpu(), xn.cpu()) and float(buf[..., :64].abs().max()) == 0
    # layout converters
    xf = torch.randn(2, 37, 9, 11, generator=g)
    nh = ops.nchw_to_nhwc(xf.cuda())
    assert torch.equal(nh.cpu(), xf.permute(0, 2, 3, 1).half())
    back = ops.nhwc_to_nchw(nh)
    assert torch.equal(back.cpu(), xf.half().float())


@pytest.mark.parametrize("act", ["mish", "leaky", "relu6", "h_swish", "swish", "relu"])
def test_activation_fwd_bwd(act):
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(4096, generator=g) * 4).requires_grad_(True)
    dy = torch.randn(4096, generator=g)
    y = _ref_act(x, act)
    y.backward(dy)
    got = ops.act_fwd(x.detach().cuda(), act).cpu()
    assert torch.allclose(got, y.detach(), rtol=1e-5, atol=1e-6)
    gx = ops.act_bwd(x.detach().cuda(), dy.cuda(), act).cpu()
    assert torch.allclose(gx, x.grad, rtol=1e-4, atol=1e-5)


def test_yolo_decode_bit_exact_indexing():
    ops = _ops()
    g = torch.Generator().manual_seed(6)
    B, na, no, ny, nx, stride = 2, 3, 85, 10, 13, 16.0
    anchors = torch.tensor([[30., 61.], [62., 45.], [59., 119.]])
    raw_nchw = torch.randn(B, na * no, ny, nx, generator=g)
    # reference semantics of YOLOLayer.forward (models.py:401-437), restated
    p = raw_nchw.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
    yv, xv = torch.meshgrid([torch.arange(ny), torch.arange(nx)], indexing="ij")
    grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2).float()
    io = p.clone()
    io[..., :2] = torch.sigmoid(io[..., :2]) + grid
    io[..., 2:4] = torch.exp(io[..., 2:4]) * (anchors / stride).view(1, na, 1, 1, 2)
    io[..., :4] *= stride
    torch.sigmoid_(io[..., 4:])
    raw = torch.zeros(B, ny, nx, 256, dtype=torch.float32, device="cuda")
    raw[..., :255] = raw_nchw.permute(0, 2, 3, 1).cuda()
    total = na * ny * nx + 7
    iobuf = torch.zeros(B, total, no, device="cuda")
    _, pg = ops.yolo_decode(raw, na, no, anchors.cuda(), stride, io=iobuf, row_offset=7)
    torch.cuda.synchronize()
    assert torch.equal(pg.cpu(), p), "p (permuted raw) must be bit exact"
    got = iobuf[:, 7:].cpu().view(B, na, ny, nx, no)
    # integer grid placement: (xy/stride - sigmoid) must round to the exact cell index
    cell = torch.round(got[..., :2] / stride - torch.sigmoid(p[..., :2]))
    assert torch.equal(cell, grid.expand_as(cell)), "grid indices must be exact"
    assert torch.allclose(got, io, rtol=1e-5, atol=1e-6)
    assert float(iobuf[:, :7].abs().max()) == 0
