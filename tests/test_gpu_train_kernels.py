"""GPU parity of the training kernels (dgrad / wgrad wgmma GEMMs, BN+activation fwd/bwd, SGD) and the
quantisation kernels against torch autograd / the oracle on identical fp16-rounded operands."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import golden, orc

pytestmark = pytest.mark.gpu


def _ops():
    from b200yolo import ops
    return ops


def _nhwc(t, dtype=torch.float16):
    return t.permute(0, 2, 3, 1).contiguous().to(dtype).cuda()


def _nchw(t):
    return t.float().permute(0, 3, 1, 2).cpu()


def conv_grads_case(B, H, W, Cin, Cout, k, stride, seed=0, accumulate=False, gdt=torch.float16):
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    pad = (k - 1) // 2
    x = torch.randn(B, Cin, H, W, generator=g).half().double().requires_grad_(True)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k)).half().double().requires_grad_(True)
    y = F.conv2d(x, w, None, stride=stride, padding=pad)
    dy = torch.randn(y.shape, generator=g).to(gdt).double()
    y.backward(dy)
    dxr, dwr = x.grad.float(), w.grad.float()
    if gdt == torch.bfloat16:   # dgrad multiplies bf16-rounded weights; wgrad keeps the fp16 activations
        wb = w.detach().float().bfloat16().double().requires_grad_(True)
        F.conv2d(x.detach().double().requires_grad_(True), wb, None, stride=stride, padding=pad)
        xx = x.detach().clone().requires_grad_(True)
        F.conv2d(xx, wb, None, stride=stride, padding=pad).backward(dy)
        dxr = xx.grad.float()
    wt = ops.pack_dgrad_weights(w.detach().float().cuda(), stride, pad, (H, W), dtype=gdt)
    dyn = _nhwc(dy.float(), gdt)
    if accumulate:
        base = torch.randn(B, Cin, H, W, generator=g).to(gdt)
        out = _nhwc(base.float(), gdt)
        dx = ops.conv2d_bwd_data(dyn, wt, (B, H, W, Cin), k, stride, pad, out=out, accumulate=True)
        dxr = dxr + base.float()
    else:
        dx = ops.conv2d_bwd_data(dyn, wt, (B, H, W, Cin), k, stride, pad)
    dw = ops.conv2d_bwd_weight(_nhwc(x.detach().float()), dyn, k, stride, pad)
    torch.cuda.synchronize()
    e_dx = (_nchw(dx) - dxr).abs().max().item() / max(dxr.pow(2).mean().sqrt().item(), 1e-6)
    dwg = dw.permute(0, 3, 1, 2).cpu()
    e_dw = (dwg - dwr).abs().max().item() / max(dwr.pow(2).mean().sqrt().item(), 1e-6)
    return e_dx, e_dw


GRAD_CASES = [
    (2, 16, 16, 64, 128, 1, 1),
    (2, 16, 16, 64, 128, 3, 1),
    (2, 20, 20, 128, 256, 3, 1),
    (2, 16, 16, 64, 128, 3, 2),     # stride-2 data gradient = 4 phase GEMMs
    (1, 26, 38, 64, 64, 3, 2),      # non-square, even
    (1, 13, 13, 64, 64, 3, 2),      # odd input size: ragged phases
    (2, 16, 16, 32, 64, 3, 1),      # Cin=32 (64B swizzle atoms)
    (2, 16, 16, 16, 32, 3, 1),      # Cin=16
    (2, 10, 10, 512, 256, 1, 1),    # yolo head sized (Cout padded to 256 by the caller)
    (2, 12, 12, 256, 512, 3, 1),    # 4 co tiles, two N=128 tiles
    (4, 40, 40, 128, 128, 3, 1),    # many k-steps -> split-K > 1
    # narrow-input 3x3 layers (Cin 32 / 64)
    (2, 24, 24, 32, 128, 3, 1),     # Cin 32, N = 128 tile
    (3, 20, 22, 32, 64, 3, 2),      # Cin 32, stride 2
    (4, 40, 40, 64, 64, 3, 1),      # Cin 64, 100 k-steps over many split-K slices
    (1, 16, 16, 32, 32, 3, 1),      # Cout 32 < tile: clipped dY columns
    (2, 16, 16, 64, 192, 3, 1),     # Cin 64, three N tiles
    (1, 9, 7, 32, 64, 3, 1),        # fewer pixels than one k-step
]


@pytest.mark.parametrize("case", GRAD_CASES, ids=[str(c) for c in GRAD_CASES])
def test_conv_bwd_data_and_weight(case):
    e_dx, e_dw = conv_grads_case(*case)
    print("\n%s dx err/rms=%.3g dw err/rms=%.3g" % (case, e_dx, e_dw))
    assert e_dx < 6e-3      # fp16 store of dx
    assert e_dw < 2e-4      # fp32 accumulate + fp32 atomics


def test_dgrad_fp16_operands_bf16_output_with_device_scale():
    """the training configuration: dZ fp16 (scaled by s), weights fp16, dX accumulated in bf16, 1/s read on device."""
    ops = _ops()
    g = torch.Generator().manual_seed(12)
    B, H, W, Cin, Cout, k, stride, pad = 2, 16, 16, 64, 128, 3, 2, 1
    w = (torch.randn(Cout, Cin, k, k, generator=g) / 24).half().double()
    sc = 64.0
    dz_true = (torch.randn(B, Cout, 8, 8, generator=g) * 1e-3)
    dz16 = (dz_true * sc).half()
    x = torch.zeros(B, Cin, H, W, dtype=torch.double, requires_grad=True)
    F.conv2d(x, w, None, stride=stride, padding=pad).backward(dz16.double() / sc)
    base = (torch.randn(B, Cin, H, W, generator=g) * 1e-2).bfloat16()
    ref = x.grad.float() + base.float()
    wt = ops.pack_dgrad_weights(w.float().cuda(), stride, pad, (H, W))
    out = _nhwc(base.float(), torch.bfloat16)
    inv = torch.tensor([1.0 / sc], device="cuda")
    ops.conv2d_bwd_data(_nhwc(dz16.float()), wt, (B, H, W, Cin), k, stride, pad, out=out, accumulate=True, inv_scale=inv)
    got = _nchw(out)
    assert (got - ref).abs().max() <= 1.5e-2 * ref.abs().max()      # bf16 store
    dw = ops.conv2d_bwd_weight(_nhwc(torch.randn(B, Cin, H, W, generator=g)), _nhwc(dz16.float()), k, stride, pad,
                               inv_scale=inv)
    assert torch.isfinite(dw).all()


def test_wgrad_concurrent_streams_match_serial():
    """Weight gradients issued on two streams at once (as the training engine does with its side stream) equal the same
    gradients computed one after the other, bit for bit: the split-K partial sums of concurrent launches never mix."""
    ops = _ops()
    g = torch.Generator().manual_seed(7)
    cases = [(4, 64, 64, 32, 64), (4, 32, 32, 64, 128), (2, 40, 40, 128, 64)]
    data = [(_nhwc(torch.randn(B, Ci, H, W, generator=g)), _nhwc(torch.randn(B, Co, H, W, generator=g)))
            for B, H, W, Ci, Co in cases]
    serial = [ops.conv2d_bwd_weight(x, dy, 3, 1, 1) for x, dy in data]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    main = torch.cuda.current_stream()
    for s in streams:
        s.wait_stream(main)
    outs = [[None] * len(data) for _ in range(4)]
    for rep in range(4):                     # interleave launches of both streams so that they overlap
        for i, (x, dy) in enumerate(data):
            with torch.cuda.stream(streams[(rep + i) % 2]):
                outs[rep][i] = ops.conv2d_bwd_weight(x, dy, 3, 1, 1)
    torch.cuda.synchronize()
    for rep in range(4):
        for i in range(len(data)):
            assert torch.equal(outs[rep][i], serial[i]), (rep, cases[i])


def test_mixed_f16_bf16_operands_are_rejected():
    ops = _ops()
    x = torch.zeros(1, 8, 8, 64, dtype=torch.float16, device="cuda")
    dy = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(AssertionError):
        ops.conv2d_bwd_weight(x, dy, 3, 1, 1)


def test_conv_bwd_data_accumulate():
    e_dx, _ = conv_grads_case(2, 16, 16, 64, 128, 3, 2, accumulate=True)
    assert e_dx < 8e-3


@pytest.mark.parametrize("gdt", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("act,C", [("leaky", 64), ("mish", 32), ("linear", 24), ("relu6", 40), ("h_swish", 72),
                                   ("mish", 512), ("leaky", 8)])
def test_bn_train_fused_passes(act, C, gdt):
    """csrc/bn_train.cu: finalize fused into the forward pass, unrolled reduce / apply passes with the parameter
    gradients emitted by the apply kernel -- against torch's training-mode batch_norm + activation under autograd
    (fp64).  Channel counts cover power-of-two and MobileNet-style (24, 40, 72) vector counts; pixel count is not a
    multiple of the unroll / block geometry."""
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    B, H, W = 3, 13, 11
    z = (torch.randn(B, C, H, W, generator=g) * 2 + 0.3).half().float()
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.2
    res = torch.randn(B, C, H, W, generator=g).half().float()
    dy = torch.randn(B, C, H, W, generator=g).to(gdt).float()
    rm, rv = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    zr = z.clone().double().requires_grad_(True)
    gr, br = gamma.clone().double().requires_grad_(True), beta.clone().double().requires_grad_(True)
    rm_r, rv_r = rm.clone().double(), rv.clone().double()
    u = F.batch_norm(zr, rm_r, rv_r, gr, br, True, 0.1, 1e-5)
    y = orc.activation(u, act) + res.double()
    y.backward(dy.double())
    zn = _nhwc(z)
    s1 = z.sum(dim=(0, 2, 3)).cuda()
    s2 = (z * z).sum(dim=(0, 2, 3)).cuda()
    rmc, rvc = rm.cuda(), rv.cuda()
    out, save = ops.bn_train_fwd(zn, s1, s2, gamma.cuda(), beta.cuda(), 1e-5, 0.1, rmc, rvc, act, residual=_nhwc(res))
    dz, dgamma, dbeta, aux = ops.bn_train_bwd(zn, _nhwc(dy, gdt), gamma.cuda(), save, act, grad_out_scale=0.5)
    torch.cuda.synchronize()
    s_dev, inv_dev = float(aux[1]), float(aux[2])
    assert s_dev > 0 and abs(s_dev * inv_dev - 1.0) < 1e-6 and float(torch.log2(aux[1])) % 1.0 == 0.0
    assert float(dz.float().abs().max()) <= 4096.0 * (1 + 2.0 ** -10)     # the 2^12 target, within one fp16 ulp
    dz = dz.float() * inv_dev
    assert (_nchw(out) - y.detach().float()).abs().max() < 6e-3
    np.testing.assert_allclose(rmc.cpu().numpy(), rm_r.float().numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(rvc.cpu().numpy(), rv_r.float().numpy(), rtol=1e-4, atol=1e-5)
    mean = z.mean(dim=(0, 2, 3))
    np.testing.assert_allclose(save[0].cpu().numpy(), mean.numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(dgamma.cpu().numpy() * 2, gr.grad.float().numpy(), rtol=2e-3, atol=2e-3)
    np.testing.assert_allclose(dbeta.cpu().numpy() * 2, br.grad.float().numpy(), rtol=2e-3, atol=2e-3)
    ref_dz = zr.grad.float()
    tol = 4e-3 if gdt == torch.float16 else 2e-2
    assert (dz.permute(0, 3, 1, 2).cpu() - ref_dz).abs().max() < tol * max(1.0, ref_dz.abs().max().item())


@pytest.mark.parametrize("case", [(64, 32, 3, 1, 1, 64), (128, 64, 3, 2, 1, 128), (255, 256, 1, 1, 0, 256),
                                  (40, 24, 1, 1, 0, 40), (96, 72, 3, 2, 1, 96), (1024, 512, 3, 1, 1, 1024)],
                         ids=lambda c: "O%d_I%d_k%d_s%d" % c[:4])
def test_multi_tensor_pack_and_unpack_bit_exact(case):
    """csrc/multi.cu: the table-driven pack (fp32 OIHW -> forward + per-phase data-gradient fp16 layouts) and unpack
    (packed fp32 weight gradients -> OIHW) must reproduce the per-layer kernels bit for bit, with several layers of
    different geometry in ONE table (tile_begin search), head padding (255 -> 256 rows) and stride-2 phases."""
    import ctypes as C
    from b200yolo import lib
    from b200yolo.lib import PackItem, UnpackItem, call, ptr, stream_ptr
    ops = _ops()
    g = torch.Generator().manual_seed(11)
    layers = [case, (32, 16, 3, 1, 1, 32), (16, 8, 1, 1, 0, 16)]
    items, uitems, keep, tiles, utiles = [], [], [], 0, 0
    for (O, I, k, s, pd, Opad) in layers:
        w = torch.randn(O, I, k, k, generator=g).cuda()
        wf = torch.full((Opad, k, k, I), 7.0, dtype=torch.float16, device="cuda")
        wd = torch.full((Opad * I * k * k,), 7.0, dtype=torch.float16, device="cuda")
        dwp = torch.randn(Opad, k, k, I, generator=g).cuda()
        dst = torch.zeros(O, I, k, k, device="cuda")
        ti = lib.raw().b2y_layout_tile_i(k)
        items.append(PackItem(w.data_ptr(), wf.data_ptr(), wd.data_ptr(), O, Opad, I, k, s, pd, tiles, I))
        tiles += ((Opad + 31) // 32) * ((I + ti - 1) // ti)
        uitems.append(UnpackItem(dwp.data_ptr(), dst.data_ptr(), O, I, k, 0, utiles, I))
        utiles += ((O + 31) // 32) * ((I + ti - 1) // ti)
        keep.append((w, wf, wd, dwp, dst))
    tab = torch.frombuffer(bytearray(bytes((PackItem * len(items))(*items))), dtype=torch.uint8).cuda()
    utab = torch.frombuffer(bytearray(bytes((UnpackItem * len(uitems))(*uitems))), dtype=torch.uint8).cuda()
    call("b2y_pack_conv_weights_multi", ptr(tab), len(items), tiles, stream_ptr())
    call("b2y_unpack_wgrad_multi", ptr(utab), len(uitems), utiles, stream_ptr())
    torch.cuda.synchronize()
    for (O, I, k, s, pd, Opad), (w, wf, wd, dwp, dst) in zip(layers, keep):
        wpad = torch.cat([w, torch.zeros(Opad - O, I, k, k, device="cuda")], 0)
        ref_f, _, _ = ops.pack_conv_weights(wpad)
        H = 16
        ref_d = ops.pack_dgrad_weights(wpad, s, pd, (H, H))
        assert torch.equal(wf, ref_f), "forward layout"
        assert torch.equal(wd, ref_d), "data-gradient layout"
        ref_u = ops.unpack_wgrad(dwp[:O].contiguous(), torch.empty(O, I, k, k, device="cuda"))
        assert torch.equal(dst, ref_u), "unpacked weight gradient"


def _sgd_grouped(p, g, buf, tiles, lr, momentum, weight_decay, grad_scale=1.0, first_step=False, ema=None,
                 ema_decay=0.0, l1_coeff=0.0):
    """One ops.sgd_grouped launch with a single parameter group; `tiles` lists (start, length, flags)."""
    from b200yolo import lib
    hp = lib.OptStep()
    hp.group[0].lr, hp.group[0].momentum, hp.group[0].weight_decay = lr, momentum, weight_decay
    hp.grad_scale, hp.l1_coeff, hp.ema_decay, hp.first_step = grad_scale, l1_coeff, ema_decay, int(first_step)
    table = torch.tensor([(s, n | (f << 32)) for s, n, f in tiles], dtype=torch.int64, device="cuda")
    _ops().sgd_grouped(p, g, buf, table, hp, ema=ema)


def _whole(n):
    """Tiles of at most OPT_TILE elements over one tensor of n elements."""
    from b200yolo import lib
    return [(s, min(lib.OPT_TILE, n - s), 0) for s in range(0, n, lib.OPT_TILE)]


def test_sgd_grouped_matches_torch():
    g = torch.Generator().manual_seed(4)
    p0 = torch.randn(10007, generator=g)
    pt = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([pt], lr=0.01, momentum=0.937, nesterov=True, weight_decay=5e-4)
    pc, buf = p0.clone().cuda(), torch.zeros(10007, device="cuda")
    for step in range(3):
        gr = torch.randn(10007, generator=g)
        pt.grad = gr.clone()
        opt.step()
        _sgd_grouped(pc, (gr * 4).cuda(), buf, _whole(10007), 0.01, 0.937, 5e-4, grad_scale=0.25,
                     first_step=(step == 0))
    np.testing.assert_allclose(pc.cpu().numpy(), pt.detach().numpy(), rtol=1e-5, atol=1e-6)


def test_fakequant_and_cos_search_match_reference():
    ops = _ops()
    gq = golden("quant_case")
    x = torch.from_numpy(gq["x"])
    cos = ops.cos_scale_search(x.cuda(), 8).cpu()
    _, sims = orc.cos_scale_search(x, 8)
    np.testing.assert_allclose(cos.numpy(), np.array(sims, dtype=np.float32), rtol=2e-6, atol=2e-6)
    assert int(torch.argmax(cos)) == int(np.argmax(gq["scale_list"]))
    scale = float(gq["scale"])
    y = ops.fakequant(x.cuda(), scale, 8).cpu()
    assert np.array_equal(y.numpy(), gq["y_train"]), "fake-quant must be bit exact"
    y2 = ops.fakequant((x * 1.7).cuda(), scale, 8).cpu()
    assert np.array_equal(y2.numpy(), gq["y_eval"])
    mm = ops.minmax(x.view(4, -1).cuda(), per_row=True).cpu()
    assert torch.equal(mm[:, 0], x.view(4, -1).min(1).values) and torch.equal(mm[:, 1], x.view(4, -1).max(1).values)
    mm = ops.minmax(x.view(4, -1).cuda(), per_row=False).cpu()
    assert float(mm[0, 0]) == float(x.min()) and float(mm[0, 1]) == float(x.max())


@pytest.mark.parametrize("gdt", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_data_movement_backward_kernels(gdt):
    """upsample / maxpool / add backward on 16-bit gradient tensors (channel-slice views included)."""
    import ctypes as C
    from b200yolo.lib import call, ptr, stream_ptr
    ops = _ops()
    g = torch.Generator().manual_seed(21)
    B, Cc, H, W = 2, 32, 6, 5
    # upsample x2: dx += window sums of dy, dy living in a wider (concat) buffer
    dyf = torch.randn(B, Cc, 2 * H, 2 * W, generator=g).to(gdt).float()
    basef = torch.randn(B, Cc, H, W, generator=g).to(gdt).float()
    wide = torch.zeros(B, 2 * H, 2 * W, Cc + 64, dtype=gdt, device="cuda")
    gy = wide[..., :Cc]
    gy.copy_(dyf.permute(0, 2, 3, 1).to(gdt))
    gx = _nhwc(basef, gdt)
    call("b2y_upsample_nearest_bwd", ptr(gy), ops._pitch(gy), ptr(gx), ops._pitch(gx), B, H, W, Cc, 2, ops._gdt(gy),
         stream_ptr())
    ref = basef + F.avg_pool2d(dyf, 2) * 4
    tol = 2e-3 if gdt == torch.float16 else 1.6e-2
    assert (_nchw(gx) - ref).abs().max() <= tol * ref.abs().max()
    # maxpool 2x2 s2 and the SPP-style 5x5 s1
    for k, s in ((2, 2), (5, 1)):
        x = torch.randn(B, Cc, 8, 8, generator=g).half().float().requires_grad_(True)
        y = F.max_pool2d(x, k, s, (k - 1) // 2)
        dy = torch.randn(y.shape, generator=g).to(gdt).float()
        y.backward(dy)
        gxm = torch.zeros(B, 8, 8, Cc, dtype=gdt, device="cuda")
        xn, dyn = _nhwc(x.detach()), _nhwc(dy, gdt)
        call("b2y_maxpool_bwd", ptr(xn), ops._pitch(xn), ptr(dyn), ops._pitch(dyn), ptr(gxm), ops._pitch(gxm), B, 8, 8,
             Cc, k, s, 0, ops._gdt(dyn), stream_ptr())
        assert (_nchw(gxm) - x.grad).abs().max() <= 4 * tol * max(1.0, x.grad.abs().max().item())
    # SPP windows over a 20 x 19 map with many tied maxima (first maximum in row-major window order wins, as in torch),
    # accumulated into a buffer that already holds another branch's gradient: the plane-in-shared-memory kernel
    for k in (5, 9, 13):
        x = (torch.randn(B, Cc, 20, 19, generator=g) * 2).round().div(2).requires_grad_(True)
        y = F.max_pool2d(x, k, 1, (k - 1) // 2)
        dy = torch.randn(y.shape, generator=g).to(gdt).float()
        y.backward(dy)
        base = torch.randn(B, Cc, 20, 19, generator=g).to(gdt).float()
        gxm = _nhwc(base, gdt)
        xn, dyn = _nhwc(x.detach()), _nhwc(dy, gdt)
        call("b2y_maxpool_bwd", ptr(xn), ops._pitch(xn), ptr(dyn), ops._pitch(dyn), ptr(gxm), ops._pitch(gxm), B, 20,
             19, Cc, k, 1, 0, ops._gdt(dyn), stream_ptr())
        want = (base + x.grad).to(gdt).float()          # one rounding of the exact fp32 sum
        assert (_nchw(gxm) - want).abs().max() <= 2.0 ** (-10 if gdt == torch.float16 else -7) * want.abs().max()
    # add (gradient accumulation into a slice)
    a = torch.randn(B, Cc, H, W, generator=g).to(gdt)
    b = torch.randn(B, Cc, H, W, generator=g).to(gdt)
    an, bn = _nhwc(a.float(), gdt), _nhwc(b.float(), gdt)
    ops.add(an, bn, out=an)
    assert torch.equal(_nchw(an), (a.float() + b.float()).to(gdt).float())
    # yolo permute^T with a device-side scale
    dp = torch.randn(B, 3, 4, 5, 85, generator=g)
    raw = torch.zeros(B, 4, 5, 256, dtype=gdt, device="cuda")
    sc = torch.tensor([8.0, 0.125], device="cuda")
    call("b2y_yolo_grad_to_raw", ptr(dp.cuda()), ptr(raw), 256, B, 3, 85, 4, 5, 1.0, ptr(sc), ops._gdt(raw),
         stream_ptr())
    want = (dp.permute(0, 2, 3, 1, 4).reshape(B, 4, 5, 255) * 8.0).to(gdt)
    assert torch.equal(raw[..., :255].cpu(), want) and float(raw[..., 255].abs().max()) == 0.0


def test_sgd_grouped_ema_matches_torch_and_model_ema():
    """SURVEY 8(f3): SGD-Nesterov + ModelEMA (utils/torch_utils.py:171-183) in one pass over the flat buffer."""
    import math
    g = torch.Generator().manual_seed(8)
    n = 20011
    p0 = torch.randn(n, generator=g)
    pt = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([pt], lr=0.01, momentum=0.937, nesterov=True, weight_decay=5e-4)
    ema_ref = p0.clone()
    pc, buf, ema = p0.clone().cuda(), torch.zeros(n, device="cuda"), p0.clone().cuda()
    for step in range(1, 4):
        gr = torch.randn(n, generator=g)
        pt.grad = gr.clone()
        opt.step()
        d = 0.9999 * (1 - math.exp(-step / 2000))
        ema_ref.mul_(d).add_(pt.detach(), alpha=1 - d)
        _sgd_grouped(pc, gr.cuda(), buf, _whole(n), 0.01, 0.937, 5e-4, first_step=(step == 1), ema=ema, ema_decay=d)
    np.testing.assert_allclose(pc.cpu().numpy(), pt.detach().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(ema.cpu().numpy(), ema_ref.numpy(), rtol=1e-5, atol=1e-6)


def test_bn_l1_tiles_match_update_bn():
    """SURVEY 8(f3): BNOptimizer.updateBN (prune_utils.py:133-138, train.py:444-445) on the L1-flagged tiles of the
    grouped optimiser, and through FlatDataParallel.set_bn_sparsity + step() on the real yolov3-tiny module tree."""
    from b200yolo import lib
    g = torch.Generator().manual_seed(3)
    n = 5000
    p = torch.randn(n, generator=g)
    p[::17] = 0.0                                           # torch.sign(0) == 0
    gr = torch.randn(n, generator=g)
    ranges = [(0, 32), (100, 1000), (4093, 907), (2000, 1)]
    want = gr.clone()
    for off, ln in ranges:
        want[off:off + ln] += 0.01 * torch.sign(p[off:off + ln])
    # the L1 ranges and the gaps between them as tiles; a first step without momentum or weight decay leaves g + L1 in buf
    cuts = sorted({0, n} | {b for off, ln in ranges for b in (off, off + ln)})
    tiles = [(a, b - a, lib.OPT_TILE_L1 if (a, b - a) in ranges else 0) for a, b in zip(cuts, cuts[1:])]
    buf = torch.full((n,), float("nan"), device="cuda")
    _sgd_grouped(p.cuda(), gr.cuda(), buf, tiles, 0.01, 0.0, 0.0, first_step=True, l1_coeff=0.01)
    assert torch.equal(buf.cpu(), want)

    from b200yolo.parallel import FlatDataParallel
    from helpers import build_model
    model = build_model("yolov3-tiny", device="cuda").train()
    ref = {n_: q.detach().clone().cpu() for n_, q in model.named_parameters()}
    dp = FlatDataParallel(model)
    prune_idx = [0, 2, 4, 6]
    s = 0.001
    dp.set_bn_sparsity(prune_idx, s)
    grads = {}
    for n_, q in model.named_parameters():
        grads[n_] = torch.randn(q.shape, generator=g) * 0.01
        q.grad.copy_(grads[n_].cuda())                      # views of the flat gradient buffer
    dp.step(lr=0.01, momentum=0.937, weight_decay=0.000484)
    bn_names = {"module_list.%d.BatchNorm2d.weight" % i for i in prune_idx}
    for n_, q in model.named_parameters():
        gref = grads[n_].clone()
        if n_ in bn_names:
            gref += s * torch.sign(ref[n_])
        wd = 0.000484 if ("Conv2d.weight" in n_ and ".bias" not in n_) else 0.0
        gref = gref + wd * ref[n_]
        want_p = ref[n_] - 0.01 * (gref + 0.937 * gref)     # first Nesterov step: buf = g
        np.testing.assert_allclose(q.detach().cpu().numpy(), want_p.numpy(), rtol=1e-5, atol=1e-7, err_msg=n_)
