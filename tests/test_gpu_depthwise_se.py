"""The depthwise convolution and squeeze-excite kernels of MobileNet-YOLOv3 (csrc/depthwise.cu) against fp64, at the
layer shapes training runs at 416 px: the fp16 forward with its batch statistics and its eval form, the data and weight
gradients, squeeze-excite forward and backward, and the fp32 versions the google-QAT graph runs.

A launch gives each CTA 256 threads; a thread owns one 8-channel vector (CV = C / 8 per pixel row) and a CTA covers
PPB = 256 // CV pixel rows, so every width but 16 and 64 (and 2048) leaves threads idle.  The grid is a grid-stride loop
over the pixels, capped at 4 CTAs per SM (1 per SM and tap for the weight gradient); squeeze-excite runs one row of
CTAs per image.  dw_launch / se_launch restate that choice, and every case asserts the geometry it was written for.

Inputs are read through a channel slice of a wider buffer whose other channels hold +-60000, outputs go to a channel
slot of a sentinel-filled buffer that must come back untouched, and every reduction over pixels is checked for
bit-identical repeats: the per-CTA partial sums go through the per-stream fp64 accumulator (common.cuh stream_acc), so
the result does not depend on the order in which CTAs finish."""
import math
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

SMS = 132          # H100 SXM; the expected grids below are for this SM count
SENTINEL = -768.0  # exact in fp16, bf16 and fp32
HUGE = 60000.0     # finite in fp16; any read of these channels shows up in the result
SMEM_LIMIT = 200 * 1024
DT = {"f16": torch.float16, "bf16": torch.bfloat16}

# yolov3-mobilenet's depthwise layers at 416 px: (channels, kernel, stride, input map)
LAYERS = [(16, 3, 1, 208), (64, 3, 2, 208), (72, 3, 1, 104), (72, 5, 2, 104), (120, 5, 1, 52), (240, 3, 2, 52),
          (200, 3, 1, 26), (184, 3, 1, 26), (480, 3, 1, 26), (672, 3, 1, 26), (672, 5, 2, 26), (960, 5, 1, 13)]
# its squeeze-excite layers: (channels, map)
SE_LAYERS = [(72, 52), (120, 52), (480, 26), (672, 26), (672, 13), (960, 13)]

# (C, k, s, H, B, expected grids: forward, data gradient, weight gradient per tap)
DwCase = namedtuple("DwCase", "C k s H B expect")
_CASES = [
    DwCase(16, 3, 1, 208, 8, (528, 528, 132)),
    DwCase(64, 3, 2, 208, 8, (528, 528, 132)),
    DwCase(72, 3, 1, 104, 8, (528, 528, 132)),
    DwCase(72, 5, 2, 104, 8, (528, 528, 132)),
    DwCase(120, 5, 1, 52, 8, (528, 528, 132)),
    DwCase(240, 3, 2, 52, 8, (528, 528, 132)),
    DwCase(200, 3, 1, 26, 8, (528, 528, 132)),
    DwCase(184, 3, 1, 26, 8, (492, 492, 132)),         # 492 CTAs: just under the cap
    DwCase(480, 3, 1, 26, 8, (528, 528, 132)),
    DwCase(672, 3, 1, 26, 8, (528, 528, 132)),
    DwCase(672, 5, 2, 26, 8, (451, 528, 132)),
    DwCase(960, 5, 1, 13, 8, (528, 528, 132)),         # 57 KB of dynamic shared memory
    DwCase(16, 3, 1, 208, 32, (528, 528, 132)),        # bench's training batch: 1.38 M pixels
    DwCase(8, 3, 1, 13, 1, (1, 1, 1)),                 # 169 pixels, one CTA of 256 rows
    DwCase(16, 3, 2, 13, 1, (1, 2, 1)),                # 49 output pixels, one CTA of 128 rows
    DwCase(2048, 5, 1, 13, 2, (338, 338, 132)),        # PPB = 1, 109 KB of dynamic shared memory
]


def _cname(c):
    return "c%d_k%ds%d_%d_b%d" % (c.C, c.k, c.s, c.H, c.B)


CASES = {_cname(c): c for c in _CASES}
LAYER_CASES = {_cname(c): c for c in _CASES if c.B == 8}


def out_hw(H, k, s):
    return (H + 2 * ((k - 1) // 2) - k) // s + 1


def dw_launch(C, k, s, H, B, sms=SMS):
    """b2y_dwconv_fwd / _bwd_data / _bwd_weight's launch: threads, grids and dynamic shared memory (square maps)"""
    CV = C // 8
    PPB = max(256 // CV, 1)
    Ho = out_hw(H, k, s)

    def grid(rows, per_sm):
        want = -(-rows // PPB)
        return max(1, min(want, sms * per_sm)), want > sms * per_sm

    fwd, fwd_capped = grid(B * Ho * Ho, 4)
    dgrad, dgrad_capped = grid(B * H * H, 4)
    wgrad, wgrad_capped = grid(B * Ho * Ho, 1)
    smem = (k * k * C * 2 + 15) // 16 * 16 + 256 * 9 * 4
    return dict(CV=CV, PPB=PPB, active=CV * PPB, fwd=fwd, fwd_capped=fwd_capped, dgrad=dgrad,
                dgrad_capped=dgrad_capped, wgrad=(wgrad, k * k), wgrad_capped=wgrad_capped, smem=smem,
                rows=B * Ho * Ho)


def se_launch(C, HW, B, sms=SMS):
    """b2y_se_fwd / _bwd's pixel-reduction grid: (CTAs per image, images)"""
    PPB = 256 // (C // 8)
    want = -(-HW // PPB)
    cap = -(-4 * sms // B)
    return dict(PPB=PPB, gx=max(1, min(want, cap)), capped=want > cap)


# ---------------------------------------------------------------------------------------------------------------
# CPU: the tables
# ---------------------------------------------------------------------------------------------------------------
def test_layer_table_matches_the_generated_cfg():
    """LAYERS / SE_LAYERS are the depthwise and SE layers of the generated yolov3-mobilenet cfg at 416 px."""
    from helpers import module_defs
    size, dw, se = 416, set(), set()
    for d in module_defs("yolov3-mobilenet"):
        t = d["type"]
        if t in ("route", "upsample", "yolo"):
            break                          # the backbone ends here: every depthwise and SE layer is before it
        if t in ("convolutional", "depthwise"):
            k, s = int(d["size"]), int(d["stride"])
            pad = (k - 1) // 2 if int(d["pad"]) else 0
            if t == "depthwise":
                assert pad == (k - 1) // 2
                dw.add((int(d["filters"]), k, s, size))
            size = (size + 2 * pad - k) // s + 1
        elif t == "se":
            se.add((int(d["filters"]), size))
    assert dw == set(LAYERS)
    assert se == set(SE_LAYERS)


def test_case_table_covers_every_launch_path():
    geo = {n: dw_launch(c.C, c.k, c.s, c.H, c.B) for n, c in CASES.items()}
    for n, c in CASES.items():
        g = geo[n]
        assert (g["fwd"], g["dgrad"], g["wgrad"][0]) == c.expect, (n, g)
    assert set(LAYER_CASES) == {_cname(DwCase(*layer, 8, None)) for layer in LAYERS}
    # idle threads: every width but 16, 64 and 2048
    assert {c.C for n, c in CASES.items() if geo[n]["active"] < 256} == {72, 120, 240, 200, 184, 480, 672, 960}
    assert all(geo[n]["active"] == 256 for n, c in CASES.items() if c.C in (8, 16, 64, 2048))
    for key in ("fwd_capped", "dgrad_capped", "wgrad_capped"):
        assert {geo[n][key] for n in CASES} == {True, False}, key
    # a map with fewer output pixels than one CTA's rows
    assert any(g["rows"] < g["PPB"] for g in geo.values())
    # dynamic shared memory above the 48 KB default (960 / k5, 2048 / k5) and up to the 200 KB limit; 2048 / k7 is over
    assert dw_launch(960, 5, 1, 13, 8)["smem"] > 48 * 1024
    assert 48 * 1024 < dw_launch(2048, 5, 1, 13, 2)["smem"] <= SMEM_LIMIT
    assert dw_launch(2048, 7, 1, 13, 2)["smem"] > SMEM_LIMIT
    assert max(g["smem"] for n, g in geo.items() if CASES[n].C < 960) <= 48 * 1024
    # squeeze-excite: capped and uncapped reductions
    se = [se_launch(C, H * H, 8) for C, H in SE_LAYERS]
    assert [s["gx"] for s in se] == [66, 66, 66, 66, 57, 66]
    assert {s["capped"] for s in se} == {True, False}


# ---------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------
def _ops():
    from b200yolo import ops
    return ops


def _seed(name):
    return zlib.crc32(name.encode()) % 10007


def _huge_buffer(g, shape, dtype):
    sign = torch.randint(0, 2, shape, generator=g, device="cuda", dtype=torch.int8)
    return (sign.to(dtype) * 2 - 1) * HUGE


def _input_view(g, B, H, W, C, dtype=torch.float16, offset=0.0):
    """channels [8, 8 + C) of a wider NHWC buffer whose other channels hold +-HUGE; returns (view, fp64 NCHW)"""
    buf = _huge_buffer(g, (B, H, W, C + 16), dtype)
    buf[..., 8:8 + C] = (torch.randn(B, H, W, C, generator=g, device="cuda") + offset).to(dtype)
    v = buf[..., 8:8 + C]
    return v, _nchw64(v)


def _output_slot(B, H, W, C, dtype, lead=8, trail=8):
    buf = torch.full((B, H, W, lead + C + trail), SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[..., lead:lead + C]


def _assert_slot_only(buf, lead, n):
    s = torch.full((), SENTINEL, dtype=buf.dtype, device=buf.device)
    assert bool((buf[..., :lead] == s).all()) and bool((buf[..., lead + n:] == s).all()), \
        "wrote outside the channel slot"


def _nchw64(t):
    return t.permute(0, 3, 1, 2).double()


def _ulp(t64, dtype):
    """one ulp of `dtype` at |t64| (its subnormal spacing below the normal range)"""
    mant, emin = {torch.float16: (10, -14), torch.bfloat16: (7, -126)}[dtype]
    return torch.exp2(torch.floor(torch.log2(t64.abs().clamp(min=2.0 ** emin))) - mant)


def _act64(y, act):
    if act == "relu6":
        return y.clamp(0.0, 6.0)
    if act == "h_swish":
        return y * (y + 3.0).clamp(0.0, 6.0) / 6.0
    return y


def _weights(g, C, k):
    """fp32 [C][1][k][k] module parameter, and the fp16-rounded fp64 copy the kernels compute with"""
    w = torch.randn(C, 1, k, k, generator=g, device="cuda") / k
    return w, w.half().double()


def _check_within(tag, got, ref, tol):
    excess = ((got - ref).abs() / tol).max().item()
    print("%s: max err %.3g of its tolerance" % (tag, excess))
    assert excess <= 1.0, "%s: error %.3g times the tolerance" % (tag, excess)


def _check_stats(tag, launch, C, M):
    """launch(s1, s2) adds the batch sums of one forward into s1, s2 and returns the fp16 z it stored.  Against fp64
    sums of that stored z (the kernel sums the rounded value): fresh sums, sums added into pre-filled buffers,
    bit-identical repeats, and bn_train_fwd's mean, invstd and running statistics."""
    ops = _ops()
    dev = "cuda"
    # the first launch, into sums twice as wide as the layer: nothing past channel C may change
    probe1 = torch.zeros(2 * C, device=dev)
    probe2 = torch.zeros(2 * C, device=dev)
    z = launch(probe1[:C], probe2[:C])
    assert bool((probe1[C:] == 0).all()) and bool((probe2[C:] == 0).all()), "sums written past channel C"
    z64 = _nchw64(z)
    ref1 = z64.sum(dim=(0, 2, 3))
    ref2 = z64.square().sum(dim=(0, 2, 3))
    # fp32 partial sums of a few hundred rows per CTA, added in fp64: 1e-5 of the sum of |terms| bounds them
    tol1 = 1e-5 * z64.abs().sum(dim=(0, 2, 3)) + 1e-30
    tol2 = 1e-5 * ref2 + 1e-30
    s1 = torch.zeros(C, device=dev)
    s2 = torch.zeros(C, device=dev)
    launch(s1, s2)
    e1 = ((s1.double() - ref1).abs() / tol1).max().item()
    e2 = ((s2.double() - ref2).abs() / tol2).max().item()

    g = torch.Generator(device=dev).manual_seed(5)
    base1 = torch.randn(C, generator=g, device=dev) * ref1.abs().max().float()
    base2 = torch.rand(C, generator=g, device=dev) * ref2.max().float()
    a1, a2 = base1.clone(), base2.clone()
    launch(a1, a2)
    b1, b2 = base1.clone(), base2.clone()
    launch(b1, b2)
    want1, want2 = base1.double() + ref1, base2.double() + ref2
    ea1 = ((a1.double() - want1).abs() / (tol1 + 2.0 ** -23 * want1.abs())).max().item()
    ea2 = ((a2.double() - want2).abs() / (tol2 + 2.0 ** -23 * want2.abs())).max().item()

    gamma = torch.rand(C, generator=g, device=dev) + 0.5
    beta = torch.randn(C, generator=g, device=dev) * 0.2
    rm = torch.randn(C, generator=g, device=dev) * 0.1
    rv = torch.rand(C, generator=g, device=dev) + 0.5
    rm0, rv0 = rm.double(), rv.double()
    _, save = ops.bn_train_fwd(z, s1, s2, gamma, beta, 1e-5, 0.1, rm, rv, "linear")
    mean = z64.mean(dim=(0, 2, 3))
    var = (z64 - mean.view(1, -1, 1, 1)).square().mean(dim=(0, 2, 3))     # two-pass
    invstd = 1.0 / torch.sqrt(var + 1e-5)
    rv_ref = 0.9 * rv0 + 0.1 * var * (M / (M - 1))
    rm_ref = 0.9 * rm0 + 0.1 * mean
    chain = dict(
        mean=((save[0].double() - mean).abs() / (mean.abs() + var.sqrt())).max().item(),
        invstd=((save[1].double() - invstd).abs() / invstd).max().item(),
        running_var=((rv.double() - rv_ref).abs() / rv_ref).max().item(),
        running_mean=((rm.double() - rm_ref).abs() / (rm_ref.abs() + 0.1 * var.sqrt())).max().item(),
        mean_over_sigma=(mean.abs() / var.sqrt()).median().item())
    print("%s: sum %.3g sq %.3g acc_sum %.3g acc_sq %.3g %s" % (tag, e1, e2, ea1, ea2, chain))
    assert e1 <= 1.0 and e2 <= 1.0, "batch sums off: %g %g (units of the tolerance)" % (e1, e2)
    assert ea1 <= 1.0 and ea2 <= 1.0, "sums do not accumulate into the pre-filled buffers: %g %g" % (ea1, ea2)
    assert torch.equal(a1, b1) and torch.equal(a2, b2), "a repeated launch gives different sums"
    assert chain["mean"] <= 1e-4 and chain["invstd"] <= 1e-4, chain
    assert chain["running_var"] <= 1e-4 and chain["running_mean"] <= 1e-4, chain
    return z64, chain


# ---------------------------------------------------------------------------------------------------------------
# forward and batch statistics
# ---------------------------------------------------------------------------------------------------------------
STATS_CASES = dict(CASES)
STATS_CASES["c72_k3s1_104_b8_mean8sigma"] = CASES["c72_k3s1_104_b8"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STATS_CASES))
def test_depthwise_forward_and_statistics_against_fp64(name):
    c = STATS_CASES[name]
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(_seed(name))
    pad = (c.k - 1) // 2
    Ho = out_hw(c.H, c.k, c.s)
    geo = dw_launch(c.C, c.k, c.s, c.H, c.B, torch.cuda.get_device_properties(0).multi_processor_count)
    assert (geo["fwd"], geo["dgrad"], geo["wgrad"][0]) == c.expect
    mean8 = name.endswith("mean8sigma")
    if mean8:
        # positive weights and a per-channel input offset that puts each channel's mean (inside the border) at 8 sigma
        w = (torch.rand(c.C, 1, c.k, c.k, generator=g, device="cuda") + 0.5) / c.k
        w16 = w.half().double()
        off = 8.0 * w16.square().sum(dim=(1, 2, 3)).sqrt() / w16.sum(dim=(1, 2, 3))
        xv, _ = _input_view(g, c.B, c.H, c.H, c.C)
        xv.add_(off.half().view(1, 1, 1, -1))
        x64 = _nchw64(xv)
    else:
        w, w16 = _weights(g, c.C, c.k)
        xv, x64 = _input_view(g, c.B, c.H, c.H, c.C)
    obuf, ov = _output_slot(c.B, Ho, Ho, c.C, torch.float16)

    def launch(s1, s2):
        ops.dwconv2d(xv, w, c.k, c.s, pad, out=ov, stats=(s1, s2))
        return ov

    _, chain = _check_stats(name, launch, c.C, c.B * Ho * Ho)
    if mean8:
        assert chain["mean_over_sigma"] > 6.0, chain
    ref = F.conv2d(x64, w16, None, stride=c.s, padding=pad, groups=c.C)
    mag = F.conv2d(x64.abs(), w16.abs(), None, stride=c.s, padding=pad, groups=c.C)
    z = _nchw64(ov)
    # one fp16 ulp, plus the fp32 accumulation of k^2 products
    _check_within(name, z, ref, _ulp(torch.maximum(ref.abs(), z.abs()), torch.float16) + c.k ** 2 * 2.0 ** -24 * mag)
    _assert_slot_only(obuf, 8, c.C)


EVAL_CASES = {"c16_k3s1_208_b8_relu6": ("c16_k3s1_208_b8", "relu6"),
              "c72_k5s2_104_b8_relu6": ("c72_k5s2_104_b8", "relu6"),
              "c240_k3s2_52_b8_h_swish": ("c240_k3s2_52_b8", "h_swish"),
              "c960_k5s1_13_b8_h_swish": ("c960_k5s1_13_b8", "h_swish")}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EVAL_CASES))
def test_depthwise_eval_forward_folded_bn_against_fp64(name):
    """the inference form: y = act(conv * scale + bias) with BatchNorm folded into scale and bias, no statistics"""
    case, act = EVAL_CASES[name]
    c = CASES[case]
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(_seed(name))
    pad = (c.k - 1) // 2
    Ho = out_hw(c.H, c.k, c.s)
    w, w16 = _weights(g, c.C, c.k)
    xv, x64 = _input_view(g, c.B, c.H, c.H, c.C)
    scale = torch.rand(c.C, generator=g, device="cuda") * 2 + 0.25
    bias = torch.randn(c.C, generator=g, device="cuda")
    obuf, ov = _output_slot(c.B, Ho, Ho, c.C, torch.float16)
    ops.dwconv2d(xv, w, c.k, c.s, pad, scale=scale, bias=bias, act=act, out=ov)
    conv = F.conv2d(x64, w16, None, stride=c.s, padding=pad, groups=c.C)
    mag = F.conv2d(x64.abs(), w16.abs(), None, stride=c.s, padding=pad, groups=c.C)
    pre = conv * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    ref = _act64(pre, act)
    y = _nchw64(ov)
    # one fp16 ulp; the fp32 sum, scale, bias and activation stay far inside 2^-20 of the magnitudes involved
    slack = 2.0 ** -20 * (mag * scale.double().view(1, -1, 1, 1) + bias.double().abs().view(1, -1, 1, 1) + pre.abs())
    _check_within(name, y, ref, _ulp(torch.maximum(ref.abs(), y.abs()), torch.float16) + slack)
    _assert_slot_only(obuf, 8, c.C)


# ---------------------------------------------------------------------------------------------------------------
# data gradient
# ---------------------------------------------------------------------------------------------------------------
# (C, k, s, H, B, dX dtype, accumulate, device inv_scale)
DgCase = namedtuple("DgCase", "C k s H B dt acc inv")
DGRAD_CASES = {
    "c16_k3s1_208_b8_f16": DgCase(16, 3, 1, 208, 8, "f16", False, False),
    "c64_k3s2_208_b8_bf16_acc_inv": DgCase(64, 3, 2, 208, 8, "bf16", True, True),
    "c72_k5s2_27_b8_f16_acc_inv": DgCase(72, 5, 2, 27, 8, "f16", True, True),
    "c120_k5s1_27_b8_bf16_inv": DgCase(120, 5, 1, 27, 8, "bf16", False, True),
    "c240_k3s2_27_b8_bf16_inv": DgCase(240, 3, 2, 27, 8, "bf16", False, True),
    "c480_k3s1_26_b8_f16_acc": DgCase(480, 3, 1, 26, 8, "f16", True, False),
    "c672_k5s2_13_b8_f16_inv": DgCase(672, 5, 2, 13, 8, "f16", False, True),
    "c960_k5s1_13_b8_bf16_acc": DgCase(960, 5, 1, 13, 8, "bf16", True, False),
    "c16_k3s2_13_b1_f16_acc_inv": DgCase(16, 3, 2, 13, 1, "f16", True, True),
    "c2048_k5s1_13_b2_f16_acc_inv": DgCase(2048, 5, 1, 13, 2, "f16", True, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DGRAD_CASES))
def test_depthwise_data_gradient_against_fp64(name):
    """dX written into (or added into) channels [16, 16 + C) of a wider sentinel-filled gradient buffer, from dz read
    through a channel slice of a wider buffer, as the training engine runs it"""
    c = DGRAD_CASES[name]
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(_seed(name))
    pad = (c.k - 1) // 2
    Ho = out_hw(c.H, c.k, c.s)
    dt = DT[c.dt]
    w, w16 = _weights(g, c.C, c.k)
    dzv, dz64 = _input_view(g, c.B, Ho, Ho, c.C)
    gbuf, dxv = _output_slot(c.B, c.H, c.H, c.C, dt, 16, 8)
    if c.acc:
        dxv.copy_(torch.randn(c.B, c.H, c.H, c.C, generator=g, device="cuda").to(dt))
    base = _nchw64(dxv) if c.acc else torch.zeros((), dtype=torch.float64, device="cuda")
    inv = torch.tensor([0.3], device="cuda") if c.inv else None
    s = float(inv.item()) if c.inv else 1.0
    ops.dwconv2d_bwd_data(dzv, w, (c.B, c.H, c.H, c.C), c.k, c.s, pad, out=dxv, accumulate=c.acc, inv_scale=inv)
    shape = (c.B, c.C, c.H, c.H)
    conv = torch.nn.grad.conv2d_input(shape, w16, dz64, stride=c.s, padding=pad, groups=c.C)
    mag = torch.nn.grad.conv2d_input(shape, w16.abs(), dz64.abs(), stride=c.s, padding=pad, groups=c.C)
    ref = base + s * conv
    got = _nchw64(dxv)
    # one ulp of the dX format, plus the fp32 sum of k^2 products and the fma with the pre-filled value
    tol = _ulp(torch.maximum(ref.abs(), got.abs()), dt) + 2.0 ** -20 * (s * mag + base.abs())
    _check_within(name, got, ref, tol)
    _assert_slot_only(gbuf, 16, c.C)


# ---------------------------------------------------------------------------------------------------------------
# weight gradient
# ---------------------------------------------------------------------------------------------------------------
ALPHA = 0.375
INV_SCALE = 0.3


def _wgrad_operands(name, c):
    g = torch.Generator(device="cuda").manual_seed(_seed(name) + 11)
    pad = (c.k - 1) // 2
    Ho = out_hw(c.H, c.k, c.s)
    xv, x64 = _input_view(g, c.B, c.H, c.H, c.C)
    dzv, dz64 = _input_view(g, c.B, Ho, Ho, c.C)
    grad = ALPHA * INV_SCALE * torch.nn.grad.conv2d_weight(x64, (c.C, 1, c.k, c.k), dz64, stride=c.s, padding=pad,
                                                           groups=c.C)
    rms = grad.square().mean().sqrt().item()
    base = torch.randn(c.C, 1, c.k, c.k, generator=g, device="cuda") * rms
    return xv, dzv, base, grad, rms


def _wgrad_launch(c, xv, dzv, base, inv):
    dw = base.clone()
    _ops().dwconv2d_bwd_weight(xv, dzv, c.k, c.s, (c.k - 1) // 2, alpha=ALPHA, dw=dw, inv_scale=inv)
    return dw


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_depthwise_weight_gradient_against_fp64(name):
    """dW added into a pre-filled gradient with alpha and the device inv_scale, as train_engine calls it; repeats give
    the same bits"""
    c = CASES[name]
    xv, dzv, base, grad, rms = _wgrad_operands(name, c)
    inv = torch.tensor([INV_SCALE], device="cuda")
    dw = _wgrad_launch(c, xv, dzv, base, inv)
    want = base.double() + grad
    err = ((dw.double() - want).abs() - 2.0 ** -24 * want.abs()).max().item()
    print("%s: err/rms %.3g" % (name, err / rms))
    assert err / rms < 2e-4, "max err %g rms %g" % (err, rms)
    assert torch.equal(dw, _wgrad_launch(c, xv, dzv, base, inv)), "a repeated launch gives a different dW"


@pytest.mark.gpu
def test_depthwise_weight_gradient_two_streams_match_serial():
    """Every layer's weight gradient issued alternately on two streams equals the serial run bit for bit: each stream
    has its own fp64 accumulator"""
    inv = torch.tensor([INV_SCALE], device="cuda")
    items = [(CASES[n],) + _wgrad_operands(n, CASES[n])[:3] for n in LAYER_CASES]
    serial = [_wgrad_launch(c, xv, dzv, base, inv) for c, xv, dzv, base in items]
    cur = torch.cuda.current_stream()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(cur)
    out = []
    for i, (c, xv, dzv, base) in enumerate(items):
        with torch.cuda.stream(streams[i % 2]):
            out.append(_wgrad_launch(c, xv, dzv, base, inv))
    for s in streams:
        cur.wait_stream(s)
    torch.cuda.synchronize()
    for n, a, b in zip(LAYER_CASES, serial, out):
        assert torch.equal(a, b), "%s: two-stream dW differs from the serial run" % n


# ---------------------------------------------------------------------------------------------------------------
# squeeze-excite
# ---------------------------------------------------------------------------------------------------------------
def _se_ref(x64, w1, w2, dy64, v_mask=None, h_mask=None):
    """fp64 squeeze-excite forward and backward (NCHW).  v_mask / h_mask: HardSigmoid and ReLU gradient masks to use
    instead of fp64's own (the kernel's branch where a value lies within rounding of the kink)"""
    HW = x64.shape[2] * x64.shape[3]
    w1, w2 = w1.double(), w2.double()
    mean = x64.mean(dim=(2, 3))
    a = mean @ w1.t()
    h = a.clamp(min=0.0)
    v = h @ w2.t()
    s = (v + 3.0).clamp(0.0, 6.0) / 6.0
    y = x64 * s[:, :, None, None]
    ds = (dy64 * x64).sum(dim=(2, 3))
    vm = ((v > -3.0) & (v < 3.0)) if v_mask is None else v_mask
    hm = (h > 0) if h_mask is None else h_mask
    dv = ds * vm.double() / 6.0
    dh = (dv @ w2) * hm.double()
    dmean = dh @ w1
    dx = dy64 * s[:, :, None, None] + (dmean / HW)[:, :, None, None]
    # magnitude bound of dmean: the same chain over |terms|
    dm_mag = ((dy64 * x64).abs().sum(dim=(2, 3)) / 6.0 @ w2.abs()) @ w1.abs()
    v_mag = (x64.abs().mean(dim=(2, 3)) @ w1.abs().t()) @ w2.abs().t()
    return dict(mean=mean, h=h, v=v, s=s, y=y, dv=dv, dh=dh, dmean=dmean, dx=dx, dw1=dh.t() @ mean, dw2=dv.t() @ h,
                dm_mag=dm_mag, v_mag=v_mag)


def _se_weights(g, C, cr, scale=2.0):
    w1 = torch.randn(cr, C, generator=g, device="cuda") / math.sqrt(C) * scale
    w2 = torch.randn(C, cr, generator=g, device="cuda") / math.sqrt(cr) * scale
    return w1, w2


def _ws_views(ws, B, C, cr):
    """b2y_se_fwd's workspace: mean [B][C] | v [B][C] | s [B][C] | h [B][cr]"""
    f = ws.reshape(-1)
    return dict(mean=f[:B * C].view(B, C), v=f[B * C:2 * B * C].view(B, C), s=f[2 * B * C:3 * B * C].view(B, C),
                h=f[3 * B * C:3 * B * C + B * cr].view(B, cr))


SE_CASES = {"c%d_%d_b8_%s" % (C, H, dt): (C, H, 8, dt)
            for (C, H), dt in zip(SE_LAYERS, ["bf16", "f16", "bf16", "f16", "f16", "bf16"])}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SE_CASES))
def test_squeeze_excite_against_fp64(name):
    """se_fwd, then se_bwd adding dX into a pre-filled slot with grad_scale on dW1 / dW2; the inputs have a non-zero
    mean so that the pooled-mean term dmean / HW of dX is well above the dX ulp"""
    C, H, B, dts = SE_CASES[name]
    ops = _ops()
    dt = DT[dts]
    cr, HW = C // 4, H * H
    grad_scale = 0.5
    g = torch.Generator(device="cuda").manual_seed(_seed(name))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    launch = se_launch(C, HW, B, sms)
    assert launch["gx"] == dict(zip(SE_LAYERS, [66, 66, 66, 66, 57, 66]))[(C, H)]
    xv, x64 = _input_view(g, B, H, H, C, offset=0.5)
    dyv, dy64 = _input_view(g, B, H, H, C, dtype=dt, offset=0.5)
    w1, w2 = _se_weights(g, C, cr)
    ybuf, yv = _output_slot(B, H, H, C, torch.float16)
    _, ws = ops.se_fwd(xv, w1, w2, out=yv)
    y2buf, yv2 = _output_slot(B, H, H, C, torch.float16)
    _, ws2 = ops.se_fwd(xv, w1, w2, out=yv2)
    assert torch.equal(ws, ws2) and torch.equal(ybuf, y2buf), "a repeated forward gives different bits"
    kv = _ws_views(ws, B, C, cr)
    ref = _se_ref(x64, w1, w2, dy64, v_mask=(kv["v"] > -3) & (kv["v"] < 3), h_mask=kv["h"] > 0)

    # the fp32 chain: the pooled sum from per-thread and per-CTA fp32 partials, two fp32 matrix-vector products
    rows = -(-HW // (launch["gx"] * launch["PPB"])) + launch["PPB"]
    e = 2.0 ** -24
    v_tol = (C + cr + rows + 8) * e * ref["v_mag"] + 1e-30
    _check_within(name + " v", kv["v"].double(), ref["v"], v_tol)
    y = _nchw64(yv)
    ytol = _ulp(torch.maximum(ref["y"].abs(), y.abs()), torch.float16) + x64.abs() * (v_tol / 6.0)[:, :, None, None]
    _check_within(name + " y", y, ref["y"], ytol)
    _assert_slot_only(ybuf, 8, C)

    def backward():
        gbuf, dxv = _output_slot(B, H, H, C, dt, 16, 8)
        dxv.copy_(torch.randn(B, H, H, C, generator=torch.Generator(device="cuda").manual_seed(3),
                              device="cuda").to(dt))
        base = _nchw64(dxv)
        wsb = ops.se_workspace(B, C, cr, "cuda")
        dw1 = torch.full_like(w1, SENTINEL)
        dw2 = torch.full_like(w2, SENTINEL)
        ops.se_bwd(xv, dyv, w1, w2, ws, dxv, accumulate=True, dw1=dw1, dw2=dw2, grad_scale=grad_scale, ws_bwd=wsb)
        return gbuf, dxv, base, dw1, dw2, wsb

    gbuf, dxv, base, dw1, dw2, wsb = backward()
    gbuf2, _, _, dw1b, dw2b, wsb2 = backward()
    assert torch.equal(gbuf, gbuf2) and torch.equal(dw1, dw1b) and torch.equal(dw2, dw2b) and torch.equal(wsb, wsb2), \
        "a repeated backward gives different bits"
    dx = _nchw64(dxv)
    want = base + ref["dx"]
    # one ulp of dX, the fp32 fma of dy * s and the pre-filled value, and the fp32 sum of dy * x feeding dmean
    # (per-thread and per-CTA fp32 partials, then two fp32 matrix-vector products)
    dm_tol = (C + cr + rows + 8) * e * ref["dm_mag"]
    tol = (_ulp(torch.maximum(want.abs(), dx.abs()), dt) + 2.0 ** -20 * (base.abs() + dy64.abs())
           + (dm_tol / HW)[:, :, None, None] + dy64.abs() * (v_tol / 6.0)[:, :, None, None])
    _check_within(name + " dx", dx, want, tol)
    # the pooled-mean term matters at this tolerance: without it dX would be off by many tolerances
    assert ((ref["dmean"].abs() / HW)[:, :, None, None] / tol).max().item() > 10.0
    _assert_slot_only(gbuf, 16, C)
    for key, got in (("dw1", dw1), ("dw2", dw2)):
        r = grad_scale * ref[key]
        e = (got.double() - r).abs().max().item() / r.abs().max().item()
        print("%s %s: max err / max %.3g" % (name, key, e))
        assert e < 2e-4, (key, e)


@pytest.mark.gpu
@pytest.mark.parametrize("dts", ["f16", "bf16"])
def test_squeeze_excite_hardsigmoid_edges(dts):
    """Channels whose pre-activation v is exactly -3 and +3 (HardSigmoid's kinks, gradient 0) and a hidden unit whose
    pre-activation is exactly 0 (ReLU's kink, gradient 0).  The input planes are constant over a 16 x 16 map and every
    value and weight is a small multiple of a power of two, so the means and both products are exact in fp32."""
    ops = _ops()
    dt = DT[dts]
    B, H, C = 4, 16, 72
    cr, HW = C // 4, H * H
    g = torch.Generator(device="cuda").manual_seed(21)
    plane = torch.randint(-32, 33, (B, 1, 1, C), generator=g, device="cuda").float() / 16
    plane[..., 0] = 3.0                                # channel 0: mean 3 in every image
    x = plane.expand(B, H, H, C).half().contiguous()
    w1 = torch.randint(-1, 2, (cr, C), generator=g, device="cuda").float() / 8
    w1[0] = 0.0
    w1[0, 0] = 1.0                                     # h[0] = 3 in every image
    w1[1] = 0.0                                        # h[1] = relu(0)
    w2 = torch.randint(-1, 2, (C, cr), generator=g, device="cuda").float() / 4
    edge_plus, edge_minus = 5, 6
    w2[edge_plus] = 0.0
    w2[edge_plus, 0] = 1.0                             # v = +3
    w2[edge_minus] = 0.0
    w2[edge_minus, 0] = -1.0                           # v = -3
    dy = (torch.randn(B, H, H, C, generator=g, device="cuda") + 0.5).to(dt)
    x64, dy64 = _nchw64(x), _nchw64(dy)
    ref = _se_ref(x64, w1, w2, dy64)
    assert bool((ref["v"][:, edge_plus] == 3).all()) and bool((ref["v"][:, edge_minus] == -3).all())
    assert bool((ref["h"][:, 1] == 0).all())

    y, ws = ops.se_fwd(x, w1, w2)
    kv = _ws_views(ws, B, C, cr)
    assert torch.equal(kv["mean"].double(), ref["mean"]), "the mean of a constant plane is exact"
    assert torch.equal(kv["v"].double(), ref["v"]) and torch.equal(kv["h"].double(), ref["h"])
    yt = _nchw64(y)
    _check_within("edges y", yt, ref["y"], _ulp(torch.maximum(yt.abs(), ref["y"].abs()), torch.float16))
    prev = torch.randn(B, H, H, C, generator=g, device="cuda").to(dt)
    dx = prev.clone()
    _, dw1, dw2 = ops.se_bwd(x, dy, w1, w2, ws, dx, accumulate=True, grad_scale=0.5)
    # the kinks contribute nothing: dW2's rows of the edge channels and dW1's row of the dead hidden unit are exact zeros
    assert bool((dw2[edge_plus] == 0).all()) and bool((dw2[edge_minus] == 0).all()), "HardSigmoid gradient at +-3"
    assert bool((dw1[1] == 0).all()), "ReLU gradient at 0"
    for key, got in (("dw1", dw1), ("dw2", dw2)):
        r = 0.5 * ref[key]
        e = (got.double() - r).abs().max().item() / r.abs().max().item()
        assert e < 1e-5, (key, e)
    want = _nchw64(prev) + ref["dx"]
    got = _nchw64(dx)
    tol = _ulp(torch.maximum(want.abs(), got.abs()), dt) + 2.0 ** -20 * (_nchw64(prev).abs() + dy64.abs()) + \
        (1e-5 * ref["dm_mag"] / HW)[:, :, None, None]
    _check_within("edges dx", got, want, tol)


# ---------------------------------------------------------------------------------------------------------------
# fp32 versions (the google-QAT graph's float depthwise blocks and SE layers)
# ---------------------------------------------------------------------------------------------------------------
def _f32_dw(x, w, dz, k, s):
    from b200yolo import qat
    from b200yolo.lib import call, ptr, stream_ptr
    import ctypes
    C = x.shape[3]
    d, shape = qat._dw_desc(x, C, k, s, (k - 1) // 2)
    z = torch.full(shape, SENTINEL, device="cuda")
    call("b2y_dwconv_fwd_f32", ctypes.byref(d), ptr(x), ptr(w), None, ptr(z), stream_ptr())
    dx = torch.full_like(x, SENTINEL)
    dw = torch.full_like(w, SENTINEL)
    call("b2y_dwconv_bwd_f32", ctypes.byref(d), ptr(x), ptr(dz), ptr(w), ptr(dx), ptr(dw), stream_ptr())
    return z, dx, dw


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LAYER_CASES))
def test_depthwise_f32_against_fp64(name):
    c = LAYER_CASES[name]
    g = torch.Generator(device="cuda").manual_seed(_seed(name) + 5)
    pad = (c.k - 1) // 2
    Ho = out_hw(c.H, c.k, c.s)
    x = torch.randn(c.B, c.H, c.H, c.C, generator=g, device="cuda")
    dz = torch.randn(c.B, Ho, Ho, c.C, generator=g, device="cuda")
    w = torch.randn(c.C, 1, c.k, c.k, generator=g, device="cuda") / c.k
    z, dx, dw = _f32_dw(x, w, dz, c.k, c.s)
    z2, dx2, dw2 = _f32_dw(x, w, dz, c.k, c.s)
    assert torch.equal(z, z2) and torch.equal(dx, dx2) and torch.equal(dw, dw2), "a repeat gives different bits"
    x64, dz64, w64 = _nchw64(x), _nchw64(dz), w.double()
    e = 2.0 ** -24
    ref = F.conv2d(x64, w64, None, stride=c.s, padding=pad, groups=c.C)
    mag = F.conv2d(x64.abs(), w64.abs(), None, stride=c.s, padding=pad, groups=c.C)
    _check_within(name + " z", _nchw64(z), ref, c.k ** 2 * e * mag + 1e-30)
    shape = (c.B, c.C, c.H, c.H)
    ref = torch.nn.grad.conv2d_input(shape, w64, dz64, stride=c.s, padding=pad, groups=c.C)
    mag = torch.nn.grad.conv2d_input(shape, w64.abs(), dz64.abs(), stride=c.s, padding=pad, groups=c.C)
    _check_within(name + " dx", _nchw64(dx), ref, c.k ** 2 * e * mag + 1e-30)
    ref = torch.nn.grad.conv2d_weight(x64, (c.C, 1, c.k, c.k), dz64, stride=c.s, padding=pad, groups=c.C)
    mag = torch.nn.grad.conv2d_weight(x64.abs(), (c.C, 1, c.k, c.k), dz64.abs(), stride=c.s, padding=pad, groups=c.C)
    # each product rounded to fp32, summed in fp64, the total rounded to fp32
    _check_within(name + " dw", dw.double(), ref, 2 * e * mag + e * ref.abs() + 1e-30)


@pytest.mark.gpu
@pytest.mark.parametrize("C,H", SE_LAYERS)
def test_squeeze_excite_f32_against_fp64(C, H):
    from b200yolo.lib import call, ptr, stream_ptr
    B, cr, HW = 8, C // 4, H * H
    g = torch.Generator(device="cuda").manual_seed(C * 100 + H)
    x = torch.randn(B, H, H, C, generator=g, device="cuda") + 0.5
    dy = torch.randn(B, H, H, C, generator=g, device="cuda") + 0.5
    w1, w2 = _se_weights(g, C, cr)

    def run():
        y = torch.full_like(x, SENTINEL)
        ws = torch.empty(B * (3 * C + cr), device="cuda")
        call("b2y_se_fwd_f32", ptr(x), ptr(w1), ptr(w2), ptr(y), B, HW, C, cr, ptr(ws), stream_ptr())
        dx = torch.full_like(x, SENTINEL)
        dw1, dw2 = torch.full_like(w1, SENTINEL), torch.full_like(w2, SENTINEL)
        wsb = torch.empty(B * (3 * C + cr), device="cuda")
        call("b2y_se_bwd_f32", ptr(x), ptr(dy), ptr(w1), ptr(w2), ptr(ws), ptr(wsb), ptr(dx), ptr(dw1), ptr(dw2), B,
             HW, C, cr, stream_ptr())
        return y, ws, dx, dw1, dw2

    out = run()
    for a, b in zip(out, run()):
        assert torch.equal(a, b), "a repeat gives different bits"
    y, ws, dx, dw1, dw2 = out
    kv = _ws_views(ws, B, C, cr)
    x64, dy64 = _nchw64(x), _nchw64(dy)
    ref = _se_ref(x64, w1, w2, dy64, v_mask=(kv["v"] > -3) & (kv["v"] < 3), h_mask=kv["h"] > 0)
    e = 2.0 ** -24
    # two fp32 matrix-vector products over C and C / 4 terms
    v_tol = (C + cr + 4) * e * ref["v_mag"] + 1e-30
    tag = "f32 c%d_%d" % (C, H)
    _check_within(tag + " v", kv["v"].double(), ref["v"], v_tol)
    _check_within(tag + " y", _nchw64(y), ref["y"], 2 * e * ref["y"].abs() + x64.abs() * (v_tol / 6)[:, :, None, None])
    dm_tol = (C + cr + 8) * e * ref["dm_mag"]
    tol = 2 * e * ref["dx"].abs() + dy64.abs() * (v_tol / 6)[:, :, None, None] + (dm_tol / HW)[:, :, None, None] + 1e-30
    _check_within(tag + " dx", _nchw64(dx), ref["dx"], tol)
    for key, got in (("dw1", dw1), ("dw2", dw2)):
        r = ref[key]
        err = (got.double() - r).abs().max().item() / r.abs().max().item()
        print("%s %s: max err / max %.3g" % (tag, key, err))
        assert err < 5e-5, (key, err)


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_depthwise_se_refusals_are_errors():
    """Launches the kernels cannot run are B2YError, never silent output: channels not a multiple of 8, a pixel pitch
    not a multiple of 8, and weights that do not fit in 200 KB of shared memory (2048 channels, k = 7; k = 5 runs)."""
    from b200yolo.lib import B2YError
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(4)
    dev = "cuda"
    x20 = torch.randn(2, 13, 13, 20, generator=g, device=dev).half()
    w20 = torch.randn(20, 1, 3, 3, generator=g, device=dev)
    with pytest.raises(B2YError):
        ops.dwconv2d(x20, w20, 3, 1, 1)
    with pytest.raises(B2YError):
        ops.dwconv2d_bwd_data(x20, w20, (2, 13, 13, 20), 3, 1, 1)
    with pytest.raises(B2YError):
        ops.dwconv2d_bwd_weight(x20, x20, 3, 1, 1)
    with pytest.raises(B2YError):
        ops.se_fwd(x20, torch.randn(5, 20, device=dev), torch.randn(20, 5, device=dev))
    # 16 channels at a pixel pitch of 36
    x36 = torch.randn(2, 13, 13, 36, generator=g, device=dev).half()[..., :16]
    w16 = torch.randn(16, 1, 3, 3, generator=g, device=dev)
    with pytest.raises(B2YError):
        ops.dwconv2d(x36, w16, 3, 1, 1)
    with pytest.raises(B2YError):
        ops.dwconv2d_bwd_data(x36, w16, (2, 13, 13, 16), 3, 1, 1)
    with pytest.raises(B2YError):
        ops.dwconv2d_bwd_weight(x36, x36, 3, 1, 1)
    with pytest.raises(B2YError):
        ops.se_fwd(x36, torch.randn(4, 16, device=dev), torch.randn(16, 4, device=dev))
    # shared memory: k = 5 fits, k = 7 does not
    x2048 = torch.randn(1, 9, 9, 2048, generator=g, device=dev).half()
    ops.dwconv2d(x2048, torch.randn(2048, 1, 5, 5, generator=g, device=dev), 5, 1, 2)
    w7 = torch.randn(2048, 1, 7, 7, generator=g, device=dev)
    with pytest.raises(B2YError):
        ops.dwconv2d(x2048, w7, 7, 1, 3)
    with pytest.raises(B2YError):
        ops.dwconv2d_bwd_data(x2048, w7, (1, 9, 9, 2048), 7, 1, 3)
    torch.cuda.synchronize()
