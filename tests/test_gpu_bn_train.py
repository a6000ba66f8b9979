"""The training BatchNorm kernels against fp64: the fp16 forward and backward passes of every conv layer
(csrc/bn_train.cu: b2y_bn_train_fwd, b2y_bn_train_bwd_reduce, b2y_bn_train_bwd_apply), the per-channel gradient reduce
of the bias heads (csrc/train.cu: b2y_bn_act_bwd_reduce, its "v2" and generic paths) and the fp32 BatchNorm of the
google-QAT depthwise blocks (b2y_bn_f32_fwd / b2y_bn_f32_bwd).

The fp16 passes give each CTA 256 threads; a thread owns one 8-channel vector (CV = C / 8) and a CTA covers
PPB = 256 // CV pixel rows, so T = CV * PPB threads work and the rest idle (C 24 -> 255, C 1280 -> PPB 1 and 160).
The grid is one wave of 2 CTAs per SM at most; each thread walks the pixels with stride grid * PPB, U = 4 rows per
iteration of its loop, so a layer takes `sweeps` iterations and the last one is partial unless pixels is a multiple of
grid * PPB * U.  bn_launch restates that choice and every case asserts the geometry it was written for.

The references are torch's training-mode F.batch_norm (momentum 0.1, eps 1e-5) and the oracle's activation under
autograd, in fp64, on the same fp16 / bf16-rounded operands.  Inputs are read through channel slices of wider buffers
whose other channels hold +-60000, outputs go to channel slots of sentinel-filled buffers that must come back untouched,
and every reduction must repeat bit for bit, also when launches alternate between two streams."""
import math
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from helpers import orc

SMS = 132              # H100 SXM; the expected grids below are for this SM count
U = 4                  # rows per thread and loop iteration
SENTINEL = -768.0      # exact in fp16, bf16 and fp32
HUGE = 60000.0         # finite in fp16 and bf16; any read of these channels shows up in the result
EPS, MOMENTUM, SLOPE = 1e-5, 0.1, 0.1
ACTS = ["leaky", "mish", "linear", "relu", "relu6", "h_swish", "swish"]
KINKS = {"leaky": (0.0,), "relu": (0.0,), "relu6": (0.0, 6.0), "h_swish": (-3.0, 3.0)}
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
DZ_TARGET = 4096.0 * (1 + 2.0 ** -10)   # s maps the bound on max|dz| to 2^12; one fp16 ulp of rounding above it

# (B, H, W, C, activation, expected (CV, PPB, T, grid, sweeps, pixels in the last sweep or 0 when it is full))
Case = namedtuple("Case", "B H W C act expect")
_CASES = {
    "c8_2x52x52": Case(2, 52, 52, 8, "leaky", (1, 256, 256, 22, 1, 5408)),              # CV 1, uncapped grid
    "c24_8x104x104": Case(8, 104, 104, 24, "linear", (3, 85, 255, 264, 1, 86528)),      # one idle thread
    "c72_8x52x52": Case(8, 52, 52, 72, "h_swish", (9, 28, 252, 264, 1, 21632)),
    "c1280_8x13x13": Case(8, 13, 13, 1280, "leaky", (160, 1, 160, 264, 2, 296)),        # PPB 1, reduce loops twice
    "c2048_2x13x13": Case(2, 13, 13, 2048, "mish", (256, 1, 256, 264, 1, 338)),         # the widest layer
    "c64_1x1x1": Case(1, 1, 1, 64, "leaky", (8, 32, 256, 1, 1, 1)),                     # a single pixel
    "c64_8x64x66": Case(8, 64, 66, 64, "leaky", (8, 32, 256, 264, 1, 0)),               # exactly one full sweep
    "c64_8x320x320": Case(8, 320, 320, 64, "mish", (8, 32, 256, 264, 25, 8192)),        # yolov4 640, 320x320
    "c32_8x640x640": Case(8, 640, 640, 32, "mish", (4, 64, 256, 264, 49, 32768)),       # yolov4 640, the stem
    # MobileNet widths (yolov3-mobilenet at 416 px)
    "c16_8x208x208": Case(8, 208, 208, 16, "relu6", (2, 128, 256, 264, 3, 75776)),
    "c40_8x52x52": Case(8, 52, 52, 40, "h_swish", (5, 51, 255, 264, 1, 21632)),
    "c120_8x52x52": Case(8, 52, 52, 120, "relu6", (15, 17, 255, 264, 2, 3680)),
    "c200_8x26x26": Case(8, 26, 26, 200, "h_swish", (25, 10, 250, 264, 1, 5408)),
    "c480_8x26x26": Case(8, 26, 26, 480, "relu6", (60, 4, 240, 264, 2, 1184)),
    "c960_2x13x13": Case(2, 13, 13, 960, "h_swish", (120, 2, 240, 169, 1, 338)),
}
CASES = dict(_CASES)
# the backward's activation sweep: all seven, at an idle-thread width
ACT_CASES = {"c40_8x26x26_%s" % a: Case(8, 26, 26, 40, a, (5, 51, 255, 107, 1, 5408)) for a in ACTS}


def bn_launch(C, pixels, sms=SMS):
    """b2y_bn_train_fwd / _bwd_reduce / _bwd_apply's launch (csrc/bn_train.cu geo_for, wave_grid)"""
    CV = C // 8
    PPB = 256 // CV
    want = -(-pixels // PPB)
    grid = max(1, min(want, 2 * sms))
    sweep = grid * PPB * U
    return dict(CV=CV, PPB=PPB, T=CV * PPB, grid=grid, capped=want > 2 * sms, sweeps=-(-pixels // sweep),
                tail=pixels % sweep, reduce_passes=-(-CV * 16 // 256))


def _geo(c, sms=SMS):
    g = bn_launch(c.C, c.B * c.H * c.W, sms)
    return (g["CV"], g["PPB"], g["T"], g["grid"], g["sweeps"], g["tail"])


# ---------------------------------------------------------------------------------------------------------------
# CPU: the table
# ---------------------------------------------------------------------------------------------------------------
def test_case_table_covers_every_launch_geometry():
    every = dict(CASES, **ACT_CASES)
    for n, c in every.items():
        assert _geo(c) == c.expect, (n, _geo(c))
    geo = {n: bn_launch(c.C, c.B * c.H * c.W) for n, c in CASES.items()}
    assert any(g["CV"] == 1 for g in geo.values())
    Ts = {c.C: geo[n]["T"] for n, c in CASES.items()}
    assert Ts[24] == 255 and Ts[72] == 252 and Ts[1280] == 160
    assert geo["c1280_8x13x13"]["PPB"] == 1 and geo["c1280_8x13x13"]["reduce_passes"] > 1   # CV * 16 > 256
    assert max(c.C for c in CASES.values()) == 2048
    assert {g["capped"] for g in geo.values()} == {True, False}
    assert any(c.B * c.H * c.W == 1 for c in CASES.values())
    # multi-sweep layers with a partial last sweep, and a layer whose last sweep is full
    assert any(g["sweeps"] > 1 and g["tail"] for g in geo.values())
    assert any(g["tail"] == 0 for g in geo.values())
    # yolov4 at 640 px, batch 8: a 320x320 layer at C 64 and the full-resolution stem at C 32
    assert any((c.B, c.H, c.W, c.C) == (8, 320, 320, 64) for c in CASES.values())
    assert any((c.B, c.H, c.W, c.C) == (8, 640, 640, 32) for c in CASES.values())
    # MobileNet's widths with its activations
    mb = {c.C for c in CASES.values() if c.act in ("relu6", "h_swish")}
    assert {16, 40, 72, 120, 200, 480, 960} <= mb
    assert {c.act for c in CASES.values() if c.C in (16, 40, 72, 120, 200, 480, 960)} == {"relu6", "h_swish"}
    assert {c.act for c in ACT_CASES.values()} == set(ACTS)


# ---------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------
def _lib():
    from b200yolo import lib, ops
    return lib, ops


def _seed(name):
    return zlib.crc32(name.encode()) % 10007


def _huge_buffer(g, shape, dtype):
    sign = torch.randint(0, 2, shape, generator=g, device="cuda", dtype=torch.int8)
    return (sign.to(dtype) * 2 - 1) * HUGE


def _slice_of(g, values, dtype, lead=8, trail=16):
    """values (NHWC) copied into channels [lead, lead + C) of a wider buffer whose other channels hold +-HUGE"""
    B, H, W, C = values.shape
    buf = _huge_buffer(g, (B, H, W, lead + C + trail), dtype)
    buf[..., lead:lead + C] = values.to(dtype)
    return buf[..., lead:lead + C]


def _output_slot(B, H, W, C, dtype, lead=8, trail=8):
    buf = torch.full((B, H, W, lead + C + trail), SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[..., lead:lead + C]


def _assert_slot_only(buf, lead, n):
    s = torch.full((), SENTINEL, dtype=buf.dtype, device=buf.device)
    assert bool((buf[..., :lead] == s).all()) and bool((buf[..., lead + n:] == s).all()), \
        "wrote outside the channel slot"


def _nchw64(t):
    return t.permute(0, 3, 1, 2).double()


def _ch(v):
    return v.view(1, -1, 1, 1)


def _ulp16(t64):
    """one fp16 ulp at |t64| (its subnormal spacing below the normal range)"""
    return torch.exp2(torch.floor(torch.log2(t64.abs().clamp(min=2.0 ** -14))) - 10)


def _check_within(tag, got, ref, tol, mask=None):
    err = (got - ref).abs() / tol
    if mask is not None:
        err = err * mask
    excess = err.max().item()
    print("%s: max err %.3g of its tolerance" % (tag, excess))
    assert excess <= 1.0, "%s: error %.3g times the tolerance" % (tag, excess)
    return excess


def _near_kink(u64, act, scale):
    """elements whose pre-activation lies so close to a kink (but not on it) that fp32 rounding of z*scale+shift may
    pick the other branch: their derivative is not decided by the formula under test"""
    m = torch.zeros_like(u64, dtype=torch.bool)
    for k in KINKS.get(act, ()):
        d = (u64 - k).abs()
        m |= (d > 0) & (d <= 2.0 ** -18 * scale)
    return m


def _ref_bn(z64, gamma, beta, rm, rv, act, dy64=None, res64=None, training=True):
    """fp64 training-mode BatchNorm + activation under autograd: returns dict(y, u, du, dz, dgamma, dbeta, mean, var,
    rm, rv).  A one-pixel batch, which torch refuses in training, uses the same formulas (variance 0, the running
    variance updated with it as the kernel does)."""
    z = z64.detach().clone().requires_grad_(dy64 is not None)
    g = gamma.double().detach().clone().requires_grad_(dy64 is not None)
    b = beta.double().detach().clone().requires_grad_(dy64 is not None)
    rm64, rv64 = rm.double().clone(), rv.double().clone()
    N = z64.numel() // z64.shape[1]
    mean = z64.mean(dim=(0, 2, 3))
    var = (z64 - _ch(mean)).square().mean(dim=(0, 2, 3))
    if not training or N > 1:
        u = F.batch_norm(z, rm64, rv64, g, b, training, MOMENTUM, EPS)
    else:
        zm = z.mean(dim=(0, 2, 3), keepdim=True)
        u = (z - zm) / torch.sqrt((z - zm).square().mean(dim=(0, 2, 3), keepdim=True) + EPS) * _ch(g) + _ch(b)
        rm64 = (1 - MOMENTUM) * rm64 + MOMENTUM * mean
        rv64 = (1 - MOMENTUM) * rv64 + MOMENTUM * var
    u.retain_grad() if dy64 is not None else None
    y = orc.activation(u, act, SLOPE)
    if res64 is not None:
        y = y + res64
    out = dict(y=y.detach(), u=u.detach(), mean=mean, var=var, rm=rm64, rv=rv64)
    if dy64 is not None:
        y.backward(dy64)
        out.update(du=u.grad.detach(), dz=z.grad.detach(), dgamma=g.grad.detach(), dbeta=b.grad.detach())
    return out


def _stat_sums(z64):
    """the conv epilogue's fp32 channel sums of z and z^2"""
    return z64.sum(dim=(0, 2, 3)).float(), z64.square().sum(dim=(0, 2, 3)).float()


def _fwd(zv, s1, s2, gamma, beta, rm, rv, act, res=None, out=None, save=None):
    lib, ops = _lib()
    B, H, W, C = zv.shape
    n = B * H * W
    if save is None:
        save = torch.empty((4, C), dtype=torch.float32, device="cuda")
    lib.call("b2y_bn_train_fwd", lib.ptr(zv), ops._pitch(zv), lib.ptr(s1), lib.ptr(s2), n, lib.ptr(gamma),
             lib.ptr(beta), EPS, MOMENTUM, lib.ptr(rm), lib.ptr(rv), lib.ptr(save), lib.ptr(res),
             ops._pitch(res) if res is not None else 0, lib.ptr(out), ops._pitch(out), n, C, lib.ACT[act], SLOPE,
             lib.stream_ptr())
    return save


def _bwd(zv, dyv, gamma, save, act, dzv, gos, aux_in=None):
    """TrainPlan._conv_backward's sequence: the reduce into zeroed sums and a zeroed 4-float aux row, then the apply
    with scale_out = aux[1:3]; returns (sums, aux, dgamma, dbeta)"""
    lib, ops = _lib()
    B, H, W, C = zv.shape
    n = B * H * W
    sums = torch.zeros((2, C), dtype=torch.float32, device="cuda")
    aux = torch.zeros(4, dtype=torch.float32, device="cuda")
    dgamma = torch.full((C,), SENTINEL, dtype=torch.float32, device="cuda")
    dbeta = torch.full((C,), SENTINEL, dtype=torch.float32, device="cuda")
    a = lib.ACT[act]
    lib.call("b2y_bn_train_bwd_reduce", lib.ptr(zv), ops._pitch(zv), lib.ptr(dyv), ops._pitch(dyv), lib.ptr(save),
             lib.ptr(sums), lib.ptr(aux), n, C, a, SLOPE, ops._gdt(dyv), lib.stream_ptr())
    import ctypes
    lib.call("b2y_bn_train_bwd_apply", lib.ptr(zv), ops._pitch(zv), lib.ptr(dyv), ops._pitch(dyv), lib.ptr(gamma),
             lib.ptr(save), lib.ptr(sums), lib.ptr(dzv), ops._pitch(dzv), n, C, a, SLOPE, ops._gdt(dyv), lib.ptr(aux),
             ctypes.c_void_p(aux.data_ptr() + 4), lib.ptr(dgamma), lib.ptr(dbeta), float(gos), lib.stream_ptr())
    return sums, aux, dgamma, dbeta


def _params(g, C):
    gamma = torch.rand(C, generator=g, device="cuda") + 0.5
    beta = torch.randn(C, generator=g, device="cuda") * 0.5
    rm = torch.randn(C, generator=g, device="cuda") * 0.1
    rv = torch.rand(C, generator=g, device="cuda") + 0.5
    return gamma, beta, rm, rv


# ---------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------
MEAN_SIGMAS = (0.0, 8.0, 32.0)    # channel c has mean MEAN_SIGMAS[c % 3] standard deviations


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_bn_train_forward_against_fp64(name):
    """y with and without a residual, save (mean, invstd, scale, shift) and the running statistics, with channel means
    of 0, 8 and 32 standard deviations.

    The statistics are fp32: var = s2/N - mean^2 loses about (mean/sigma)^2 * 2^-24 of the variance to cancellation
    (fp32 rounding of s2, of s2/N and of mean^2, each of size mean^2 + sigma^2).  The tolerance of the variance is
    e_var = 2^-24 * (4 + 8 (mean/sigma)^2) relative, invstd gets half of it plus two roundings, and y one fp16 ulp
    plus what those errors move z*scale+shift by (times 1.5, the steepest slope of the activations)."""
    c = CASES[name]
    lib, ops = _lib()
    B, H, W, C = c.B, c.H, c.W, c.C
    N = B * H * W
    assert _geo(c, torch.cuda.get_device_properties(0).multi_processor_count) == c.expect
    g = torch.Generator(device="cuda").manual_seed(_seed(name))
    sigma = torch.rand(C, generator=g, device="cuda") * 1.5 + 0.5
    ms = torch.tensor([MEAN_SIGMAS[i % 3] for i in range(C)], device="cuda")
    z16 = (torch.randn(B, H, W, C, generator=g, device="cuda") * sigma + ms * sigma).half()
    zv = _slice_of(g, z16, torch.float16)
    res16 = torch.randn(B, H, W, C, generator=g, device="cuda").half()
    resv = _slice_of(g, res16, torch.float16, lead=16, trail=8)
    z64 = _nchw64(z16)
    s1, s2 = _stat_sums(z64)
    gamma, beta, rm0, rv0 = _params(g, C)

    worst = {}
    for with_res in (False, True):
        rm, rv = rm0.clone(), rv0.clone()
        ybuf, yv = _output_slot(B, H, W, C, torch.float16)
        save = _fwd(zv, s1, s2, gamma, beta, rm, rv, c.act, res=resv if with_res else None, out=yv)
        ref = _ref_bn(z64, gamma, beta, rm0, rv0, c.act, res64=_nchw64(res16) if with_res else None)
        mean, var = ref["mean"], ref["var"]
        invstd = 1.0 / torch.sqrt(var + EPS)
        r = (mean.abs() / var.sqrt().clamp(min=1e-30)).clamp(max=1e6)
        e_var = 2.0 ** -24 * (4 + 8 * r.square()) * var / (var + EPS) + 2.0 ** -24
        e_inv = e_var / 2 + 2.0 ** -22
        e_mean = 2.0 ** -22 * mean.abs() + 2.0 ** -30 * var.sqrt()
        g64, b64 = gamma.double(), beta.double()
        sc = g64 * invstd
        sh = b64 - mean * sc
        _check_within(name + " mean", save[0].double(), mean, e_mean)
        _check_within(name + " invstd", save[1].double(), invstd, e_inv * invstd)
        _check_within(name + " scale", save[2].double(), sc, (e_inv + 2.0 ** -23) * sc.abs())
        _check_within(name + " shift", save[3].double(), sh,
                      mean.abs() * sc.abs() * (e_inv + 2.0 ** -21) + sc.abs() * e_mean + 2.0 ** -23 * b64.abs() + 1e-30)
        rm_ref, rv_ref = ref["rm"], ref["rv"]
        _check_within(name + " running mean", rm.double(), rm_ref,
                      MOMENTUM * e_mean + 2.0 ** -22 * (rm0.double().abs() + MOMENTUM * mean.abs()) + 1e-30)
        _check_within(name + " running var", rv.double(), rv_ref,
                      MOMENTUM * var * (e_var + 2.0 ** -21) * (N / max(N - 1, 1)) + 2.0 ** -22 * rv_ref.abs())
        # per channel class: the measured invstd error against the cancellation estimate
        for k, m in enumerate(MEAN_SIGMAS):
            sel = torch.arange(C, device="cuda") % 3 == k
            if bool(sel.any()):
                e = ((save[1].double() - invstd).abs() / invstd)[sel].max().item()
                worst["invstd rel err at %g sigma" % m] = max(worst.get("invstd rel err at %g sigma" % m, 0.0), e)
        y = _nchw64(yv)
        yref = ref["y"]
        z64c = z64
        xh = (z64c - _ch(mean)) * _ch(invstd)
        du_pos = 1.5 * (_ch(g64.abs()) * xh.abs() * _ch(e_inv) + _ch(sc.abs() * e_mean)
                        + 2.0 ** -22 * (z64c.abs() * _ch(sc.abs()) + _ch(sh.abs() + b64.abs())))
        tol = _ulp16(torch.maximum(y.abs(), yref.abs())) + du_pos
        mask = ~_near_kink(ref["u"], c.act, z64c.abs() * _ch(sc.abs()) + _ch(sh.abs()) + 1.0)
        _check_within(name + (" y+res" if with_res else " y"), y, yref, tol, mask.double())
        _assert_slot_only(ybuf, 8, C)
    print(name, worst)


# ---------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------
def _bwd_operands(name, c, gdt, g=None):
    """z (mean within a standard deviation of 0), dy in the gradient dtype, both read through channel slices as the
    training plan reads a route's gradient; the forward is run on the kernels to produce `save`"""
    B, H, W, C = c.B, c.H, c.W, c.C
    g = g or torch.Generator(device="cuda").manual_seed(_seed(name))
    sigma = torch.rand(C, generator=g, device="cuda") * 1.5 + 0.5
    mu = torch.randn(C, generator=g, device="cuda") * 0.3 * sigma
    z16 = (torch.randn(B, H, W, C, generator=g, device="cuda") * sigma + mu).half()
    dy = (torch.randn(B, H, W, C, generator=g, device="cuda") * 0.1).to(gdt)
    gamma, beta, rm, rv = _params(g, C)
    return z16, dy, gamma, beta, rm, rv


def _run_bwd_case(tag, z16, dy, gamma, beta, rm, rv, act, gos=0.25, check_ref=True, g=None):
    """forward and backward on the kernels, checked against fp64; returns the results for bit-identity checks"""
    B, H, W, C = z16.shape
    N = B * H * W
    g = g or torch.Generator(device="cuda").manual_seed(_seed(tag) + 1)
    zv = _slice_of(g, z16, torch.float16, lead=8, trail=8)
    dyv = _slice_of(g, dy, dy.dtype, lead=24, trail=8)       # a channel slice of a wider concat gradient
    z64 = _nchw64(z16)
    s1, s2 = _stat_sums(z64)
    ybuf, yv = _output_slot(B, H, W, C, torch.float16)
    save = _fwd(zv, s1, s2, gamma, beta, rm.clone(), rv.clone(), act, out=yv)
    dzbuf, dzv = _output_slot(B, H, W, C, torch.float16, lead=16, trail=8)
    sums, aux, dgamma, dbeta = _bwd(zv, dyv, gamma, save, act, dzv, gos)
    torch.cuda.synchronize()
    _assert_slot_only(dzbuf, 16, C)
    s, inv = float(aux[1]), float(aux[2])
    assert s > 0 and math.log2(s) == round(math.log2(s)), "s = %r is not a power of two" % s
    assert s * inv == 1.0, "1/s is not exact: %r * %r" % (s, inv)
    dzmax = float(dzv.float().abs().max())
    print("%s: s = 2^%d, max|dz*s| = %g, aux = %s" % (tag, round(math.log2(s)), dzmax, aux.tolist()))
    assert math.isfinite(dzmax) and dzmax <= DZ_TARGET, "max|dz*s| = %g is over the 2^12 target" % dzmax
    # the parameter gradients are the sums times grad_out_scale, rounded once
    assert torch.equal(dgamma, sums[1] * gos) and torch.equal(dbeta, sums[0] * gos)
    if check_ref:
        dy64 = _nchw64(dy)
        ref = _ref_bn(z64, gamma, beta, rm, rv, act, dy64=dy64)
        mean, var = ref["mean"], ref["var"]
        invstd = 1.0 / torch.sqrt(var + EPS)
        xh = (z64 - _ch(mean)) * _ch(invstd)
        sc64 = gamma.double() * invstd
        near = _near_kink(ref["u"], act, z64.abs() * _ch(sc64.abs()) + _ch((beta.double() - mean * sc64).abs()) + 1.0)
        # what a near-kink element may move: its du by up to 1.5 |dy|
        slack = 1.5 * dy64.abs() * near
        sl1, sl2 = slack.sum(dim=(0, 2, 3)), (slack * xh.abs()).sum(dim=(0, 2, 3))
        du = ref["du"]
        S1, S2 = du.sum(dim=(0, 2, 3)), (du * xh).sum(dim=(0, 2, 3))
        # fp32 partial sums of at most a few hundred terms per thread, added in fp64, and the fp32 mean / invstd
        t1 = du.abs().sum(dim=(0, 2, 3))
        t2 = (du * xh).abs().sum(dim=(0, 2, 3))
        tol1 = 1e-5 * t1 + sl1 + 1e-30
        tol2 = 1e-5 * (t2 + t1) + sl2 + 1e-30
        _check_within(tag + " S1", sums[0].double(), S1, tol1)
        _check_within(tag + " S2", sums[1].double(), S2, tol2)
        _check_within(tag + " dbeta", dbeta.double() / gos, ref["dbeta"], tol1 + 2.0 ** -23 * S1.abs())
        _check_within(tag + " dgamma", dgamma.double() / gos, ref["dgamma"], tol2 + 2.0 ** -23 * S2.abs())
        # aux[0] = max|du| within act_grad's __expf error (a few ulp of exp, 2^-16 relative covers it)
        dumax = du.abs().max().item()
        assert abs(float(aux[0]) - dumax) <= 2.0 ** -16 * dumax + 1.5 * float((dy64.abs() * near).max()) + 1e-30, \
            (float(aux[0]), dumax)
        # dz = (dz*s) * (1/s): one fp16 ulp of max|dz*s| plus the fp32 arithmetic of its three terms
        A = _ch((gamma.double() * invstd).abs())
        mag = (z64.abs() + _ch(mean.abs())) * _ch(sc64.abs()) + _ch(beta.double().abs())
        terms = A * (du.abs() + dy64.abs() * mag / 16 + _ch(S1.abs()) / N + xh.abs() * _ch(S2.abs()) / N)
        got = _nchw64(dzv) * inv
        tol = _ulp16(torch.tensor(dzmax, dtype=torch.float64)) * inv + 2.0 ** -16 * terms \
            + A * (_ch(tol1) + xh.abs() * _ch(tol2)) / N + 1e-30
        _check_within(tag + " dz", got, ref["dz"], tol, (~near).double())
        # aux[3] = max|xhat|
        xhmax = xh.abs().max().item()
        assert abs(float(aux[3]) - xhmax) <= 2.0 ** -18 * xhmax + 1e-30, (float(aux[3]), xhmax)
    return sums, aux, dgamma, dbeta, dzv.clone(), (zv, dyv, gamma, save, act, gos)


@pytest.mark.gpu
@pytest.mark.parametrize("gdt", list(DT))
@pytest.mark.parametrize("name", list(CASES) + list(ACT_CASES))
def test_bn_train_backward_against_fp64(name, gdt):
    """S1 / S2, dgamma and dbeta times grad_out_scale, dz * aux[2], the aux row (power-of-two s, exact 1/s, max|du|,
    max|xhat|) and the 2^12 bound on max|dz*s|; then a second launch must give the same bits"""
    c = CASES.get(name) or ACT_CASES[name]
    assert _geo(c, torch.cuda.get_device_properties(0).multi_processor_count) == c.expect
    ops_in = _bwd_operands(name, c, DT[gdt])
    sums, aux, dgamma, dbeta, dz, args = _run_bwd_case(name + "_" + gdt, *ops_in, c.act)
    zv, dyv, gamma, save, act, gos = args
    _, dz2v = _output_slot(c.B, c.H, c.W, c.C, torch.float16, lead=16, trail=8)
    sums2, aux2, dgamma2, dbeta2 = _bwd(zv, dyv, gamma, save, act, dz2v, gos)
    torch.cuda.synchronize()
    for what, a, b in (("sums", sums, sums2), ("aux", aux, aux2), ("dgamma", dgamma, dgamma2),
                       ("dbeta", dbeta, dbeta2), ("dz", dz, dz2v)):
        assert torch.equal(a, b), "a repeated launch gives a different %s" % what


@pytest.mark.gpu
@pytest.mark.parametrize("gdt", list(DT))
@pytest.mark.parametrize("act", list(KINKS))
def test_bn_train_backward_on_activation_kinks(act, gdt):
    """channels whose mean is exactly 0 (symmetric values) and whose pre-activation is exactly the kink wherever z = 0:
    u = z*scale + (beta - 0*scale) = beta, so beta = the kink puts a third of the pixels on it, in the kernel and in the
    reference alike.  The derivative there must be torch's: leaky slope at 0, relu / relu6 0 at 0 and 6, h_swish 0 at -3
    and 1 at +3."""
    C, B, H, W = 64, 8, 26, 26
    g = torch.Generator(device="cuda").manual_seed(_seed(act + gdt))
    half = torch.rand(B * H * W // 3, C, generator=g, device="cuda") * 2 + 0.25
    vals = torch.cat([half, -half, torch.zeros(B * H * W - 2 * half.shape[0], C, device="cuda")])
    perm = torch.argsort(torch.rand(vals.shape[0], generator=g, device="cuda"))
    z16 = vals[perm].view(B, H, W, C).half()
    assert bool((z16.double().sum(dim=(0, 1, 2)) == 0).all())
    kinks = KINKS[act]
    beta = torch.tensor([kinks[i % len(kinks)] for i in range(C)], device="cuda")
    gamma = torch.rand(C, generator=g, device="cuda") + 0.5
    dy = (torch.randn(B, H, W, C, generator=g, device="cuda") * 0.1).to(DT[gdt])
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    _run_bwd_case("kink_%s_%s" % (act, gdt), z16, dy, gamma, beta, rm, rv, act)


@pytest.mark.gpu
def test_bn_train_backward_edge_channels():
    """one layer with a constant channel (variance 0, invstd = 1/sqrt(eps)), a gamma = 0 channel (BatchNorm-L1 sparsity
    training leaves them) and ordinary channels; the gamma = 0 channel's dz is exactly 0"""
    C, B, H, W = 64, 8, 52, 52
    g = torch.Generator(device="cuda").manual_seed(_seed("edge"))
    z16, dy, gamma, beta, rm, rv = _bwd_operands("edge", Case(B, H, W, C, "leaky", None), torch.float16, g)
    z16[..., 0] = 1.5                       # constant: the sums are exact, so the mean is exactly 1.5 and var 0
    beta[0] = 0.5                           # leaky' = 1 on the whole constant channel
    gamma[1] = 0.0
    sums, aux, dgamma, dbeta, dz, _ = _run_bwd_case("edge", z16, dy, gamma, beta, rm, rv, "leaky", g=g)
    assert bool((dz[..., 1] == 0).all()), "gamma = 0 must give dz = 0"
    assert float(dz[..., 0].float().abs().max()) > 0


@pytest.mark.gpu
def test_bn_train_backward_zero_gradient_layer():
    """an all-zero dy gives s = 1, dz = 0 and zero parameter gradients"""
    C, B, H, W = 72, 8, 26, 26
    g = torch.Generator(device="cuda").manual_seed(_seed("zero"))
    z16, dy, gamma, beta, rm, rv = _bwd_operands("zero", Case(B, H, W, C, "mish", None), torch.float16, g)
    sums, aux, dgamma, dbeta, dz, _ = _run_bwd_case("zero", z16, torch.zeros_like(dy), gamma, beta, rm, rv, "mish",
                                                    g=g)
    assert float(aux[1]) == 1.0 and float(aux[2]) == 1.0 and float(aux[0]) == 0.0
    assert bool((dz == 0).all()) and bool((dgamma == 0).all()) and bool((dbeta == 0).all())


@pytest.mark.gpu
def test_bn_train_backward_outlier_channels_stay_finite():
    """yolov4's 320x320 layer at 640 px, batch 8 (N = 819200): channels of N(0,1) values with one pixel at 1000, so
    max|xhat| ~ 670, and dy = sign(xhat), linear, gamma = 1.  A scale bound that assumes |xhat| <= 16 picks s = 512 and
    the outlier's dz * s ~ 1.2e5 overflows fp16 to inf; the bound must hold for any xhat up to sqrt(N)."""
    C, B, H, W = 8, 8, 320, 320
    N = B * H * W
    g = torch.Generator(device="cuda").manual_seed(_seed("outlier"))
    z = torch.randn(N, C, generator=g, device="cuda")
    rows = torch.randint(0, N, (C,), generator=g, device="cuda")
    z[rows, torch.arange(C, device="cuda")] = 1000.0
    z16 = z.view(B, H, W, C).half()
    z64 = z16.double()
    xh_sign = torch.sign(z64 - z64.mean(dim=(0, 1, 2)))
    dy = xh_sign.half()
    gamma, beta = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    sums, aux, dgamma, dbeta, dz, _ = _run_bwd_case("outlier", z16, dy, gamma, beta, rm, rv, "linear", g=g)
    assert float(aux[3]) > 600


@pytest.mark.gpu
def test_bn_train_backward_two_streams_match_serial():
    """the backward of several layers issued alternately on two streams, three rounds, equals the serial run bit for
    bit: each stream's sums go through its own fp64 accumulator"""
    names = ["c8_2x52x52", "c72_8x52x52", "c1280_8x13x13", "c120_8x52x52", "c960_2x13x13"]
    items = []
    for n in names:
        z16, dy, gamma, beta, rm, rv = _bwd_operands(n, CASES[n], torch.bfloat16 if len(items) % 2 else torch.float16)
        _, _, _, _, _, args = _run_bwd_case(n, z16, dy, gamma, beta, rm, rv, CASES[n].act, check_ref=False)
        items.append(args)

    def run(args):
        zv = args[0]
        _, dzv = _output_slot(*zv.shape, torch.float16, lead=16, trail=8)
        return _bwd(*args[:5], dzv, args[5]) + (dzv,)

    serial = [run(a) for a in items]
    torch.cuda.synchronize()
    cur = torch.cuda.current_stream()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(cur)
    outs = []
    for rnd in range(3):
        for i, a in enumerate(items):
            with torch.cuda.stream(streams[(rnd + i) % 2]):
                outs.append((rnd, i, run(a)))
    for s in streams:
        cur.wait_stream(s)
    torch.cuda.synchronize()
    for rnd, i, got in outs:
        for what, a, b in zip(("sums", "aux", "dgamma", "dbeta", "dz"), serial[i], got):
            assert torch.equal(a, b), "%s round %d: two-stream %s differs from the serial run" % (names[i], rnd, what)


# ---------------------------------------------------------------------------------------------------------------
# the per-channel gradient reduce of convs without BatchNorm (bias heads): b2y_bn_act_bwd_reduce
# ---------------------------------------------------------------------------------------------------------------
def act_reduce_path(C, act):
    """csrc/train.cu bn_act_bwd_reduce_launch: the one-vector-per-thread "v2" kernel needs 256 % (C/8) == 0 and a
    compile-time activation (leaky, mish, linear); everything else takes the generic warp-strip kernel"""
    return "v2" if (C // 8 <= 256 and 256 % (C // 8) == 0 and act in ("leaky", "mish", "linear")) else "generic"


# (C, act, with dgamma / mean / invstd, expected path)
ACT_REDUCE_CASES = {
    "c256_leaky_dgamma": (256, "leaky", True, "v2"),
    "c256_mish": (256, "mish", False, "v2"),
    "c256_linear_dgamma": (256, "linear", True, "v2"),
    "c80_linear": (80, "linear", False, "generic"),          # an nc=20 head: Cpad 80
    "c320_linear_dgamma": (320, "linear", True, "generic"),  # yolov3-tiny-nc100: Cpad 320
    "c256_relu6_dgamma": (256, "relu6", True, "generic"),    # a run-time activation
}


def test_act_reduce_cases_cover_both_paths():
    for n, (C, act, _, path) in ACT_REDUCE_CASES.items():
        assert act_reduce_path(C, act) == path, n
    assert {p for *_, p in ACT_REDUCE_CASES.values()} == {"v2", "generic"}


@pytest.mark.gpu
@pytest.mark.parametrize("gdt", list(DT))
@pytest.mark.parametrize("name", list(ACT_REDUCE_CASES))
def test_bias_act_backward_reduce_against_fp64(name, gdt):
    """dbeta = sum du and dgamma = sum du*xhat (du = dy * act'(x*scale + shift)) added into pre-filled accumulators,
    x and dy read through channel slices; the ops wrapper's dbeta-only form on the same data"""
    lib, ops = _lib()
    C, act, with_g, _ = ACT_REDUCE_CASES[name]
    B, H, W = 8, 26, 26
    g = torch.Generator(device="cuda").manual_seed(_seed(name + gdt))
    x16 = (torch.randn(B, H, W, C, generator=g, device="cuda") * 2).half()
    dy = torch.randn(B, H, W, C, generator=g, device="cuda").to(DT[gdt])
    xv = _slice_of(g, x16, torch.float16)
    dyv = _slice_of(g, dy, DT[gdt], lead=16, trail=8)
    scale = torch.rand(C, generator=g, device="cuda") + 0.5
    shift = torch.randn(C, generator=g, device="cuda")
    mean = torch.randn(C, generator=g, device="cuda") * 0.5 if with_g else None
    invstd = torch.rand(C, generator=g, device="cuda") + 0.5 if with_g else None
    base_b = torch.randn(C, generator=g, device="cuda") * 100
    base_g = torch.randn(C, generator=g, device="cuda") * 100 if with_g else None
    dbeta, dgamma = base_b.clone(), base_g.clone() if with_g else None
    amax = torch.zeros(1, device="cuda")
    lib.call("b2y_bn_act_bwd_reduce", lib.ptr(xv), ops._pitch(xv), lib.ptr(dyv), ops._pitch(dyv), lib.ptr(scale),
             lib.ptr(shift), lib.ptr(mean), lib.ptr(invstd), lib.ptr(dgamma), lib.ptr(dbeta), lib.ptr(amax), B * H * W,
             C, lib.ACT[act], SLOPE, ops._gdt(dyv), lib.stream_ptr())
    x64, dy64 = _nchw64(x16), _nchw64(dy)
    u = (x64 * _ch(scale.double()) + _ch(shift.double())).requires_grad_(True)
    orc.activation(u, act, SLOPE).backward(dy64)
    du = u.grad
    near = _near_kink(u.detach(), act, u.detach().abs() + 1.0)
    slack = 1.5 * (dy64.abs() * near).sum(dim=(0, 2, 3))
    xh = (x64 - _ch(mean.double())) * _ch(invstd.double()) if with_g else x64
    want_b = base_b.double() + du.sum(dim=(0, 2, 3))
    tol_b = 1e-5 * du.abs().sum(dim=(0, 2, 3)) + slack + 2.0 ** -23 * want_b.abs()
    _check_within(name + " dbeta", dbeta.double(), want_b, tol_b)
    if with_g:
        want_g = base_g.double() + (du * xh).sum(dim=(0, 2, 3))
        tol_g = 1e-5 * (du * xh).abs().sum(dim=(0, 2, 3)) + slack * xh.abs().amax(dim=(0, 2, 3)) \
            + 2.0 ** -23 * want_g.abs()
        _check_within(name + " dgamma", dgamma.double(), want_g, tol_g)
    dumax = du.abs().max().item()
    assert abs(float(amax) - dumax) <= 2.0 ** -16 * dumax + 1.5 * float((dy64.abs() * near).max())
    # the ops wrapper (dbeta only, fresh), twice: the same bits
    d1 = ops.bias_act_bwd_reduce(xv, dyv, scale, shift, act, SLOPE)
    d2 = ops.bias_act_bwd_reduce(xv, dyv, scale, shift, act, SLOPE)
    torch.cuda.synchronize()
    assert torch.equal(d1, d2), "a repeated launch gives a different dbeta"
    _check_within(name + " dbeta fresh", d1.double(), want_b - base_b.double(), tol_b)


# ---------------------------------------------------------------------------------------------------------------
# fp32 BatchNorm of the google-QAT depthwise blocks: b2y_bn_f32_fwd / b2y_bn_f32_bwd
# ---------------------------------------------------------------------------------------------------------------
# (C, B, H, activation): MobileNet depthwise outputs at 416 px, channel counts that are not multiples of 8
F32_CASES = {"c3_8x52": (3, 8, 52, "relu6"), "c100_8x26": (100, 8, 26, "h_swish"), "c960_8x13": (960, 8, 13, "linear")}


def _f32_launch(z, dy, gamma, beta, rm, rv, training, act):
    lib, _ = _lib()
    B, H, W, C = z.shape
    n = B * H * W
    save = torch.empty((4, C), dtype=torch.float32, device="cuda")
    y = torch.empty_like(z)
    lib.call("b2y_bn_f32_fwd", lib.ptr(z), n, C, lib.ptr(gamma), lib.ptr(beta), EPS, MOMENTUM, lib.ptr(rm),
             lib.ptr(rv), int(training), lib.ptr(save), lib.ptr(y), lib.ACT[act], SLOPE, lib.stream_ptr())
    coef = torch.empty((3, C), dtype=torch.float32, device="cuda")
    dz = torch.empty_like(z)
    dgamma = torch.empty(C, dtype=torch.float32, device="cuda")
    dbeta = torch.empty_like(dgamma)
    lib.call("b2y_bn_f32_bwd", lib.ptr(z), lib.ptr(dy), n, C, lib.ptr(gamma), lib.ptr(save), int(training),
             lib.ptr(coef), lib.ptr(dz), lib.ptr(dgamma), lib.ptr(dbeta), lib.ACT[act], SLOPE, lib.stream_ptr())
    return y, save, coef, dz, dgamma, dbeta


@pytest.mark.gpu
@pytest.mark.parametrize("training", [1, 0], ids=["train", "eval"])
@pytest.mark.parametrize("name", list(F32_CASES))
def test_bn_f32_against_fp64(name, training):
    """y, the running statistics, dz, dgamma and dbeta against fp64 autograd; in eval dz is exactly
    coef[0] * du with coef[0] = fp32(gamma * invstd) and zero coefficient rows 1 and 2; a repeat gives the same bits"""
    C, B, H, act = F32_CASES[name]
    W = H
    g = torch.Generator(device="cuda").manual_seed(_seed(name) + training)
    z = torch.randn(B, H, W, C, generator=g, device="cuda") * 1.5 + 0.2
    dy = torch.randn(B, H, W, C, generator=g, device="cuda")
    gamma, beta, rm0, rv0 = _params(g, C)
    rm, rv = rm0.clone(), rv0.clone()
    y, save, coef, dz, dgamma, dbeta = _f32_launch(z, dy, gamma, beta, rm, rv, training, act)
    rm2, rv2 = rm0.clone(), rv0.clone()
    again = _f32_launch(z, dy, gamma, beta, rm2, rv2, training, act)
    torch.cuda.synchronize()
    for what, a, b in zip(("y", "save", "coef", "dz", "dgamma", "dbeta"), (y, save, coef, dz, dgamma, dbeta), again):
        assert torch.equal(a, b), "a repeated launch gives a different %s" % what
    assert torch.equal(rm, rm2) and torch.equal(rv, rv2)

    z64, dy64 = _nchw64(z), _nchw64(dy)
    ref = _ref_bn(z64, gamma, beta, rm0, rv0, act, dy64=dy64, training=bool(training))
    if training:
        mean, var = ref["mean"], ref["var"]
        _check_within(name + " running mean", rm.double(), ref["rm"], 2.0 ** -22 * (ref["rm"].abs() + mean.abs()))
        _check_within(name + " running var", rv.double(), ref["rv"], 2.0 ** -21 * ref["rv"].abs())
    else:
        mean, var = rm0.double(), rv0.double()
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0), "eval must not touch the running statistics"
    invstd = 1.0 / torch.sqrt(var + EPS)
    sc = gamma.double() * invstd
    sh = beta.double() - mean * sc
    _check_within(name + " save", save.double(), torch.stack([mean, invstd, sc, sh]),
                  2.0 ** -21 * torch.stack([mean.abs(), invstd, sc.abs(), sh.abs() + (mean * sc).abs()]) + 1e-30)
    mag = (z64.abs() + _ch(mean.abs())) * _ch(sc.abs()) + _ch(sh.abs() + beta.double().abs()) + 1e-30
    near = _near_kink(ref["u"], act, mag)
    _check_within(name + " y", _nchw64(y), ref["y"], 2.0 ** -20 * 1.5 * mag + 2.0 ** -23 * ref["y"].abs(),
                  (~near).double())
    du = ref["du"]
    slack = 1.5 * (dy64.abs() * near).sum(dim=(0, 2, 3))
    xh = (z64 - _ch(mean)) * _ch(invstd)
    # fixed-order double sums of fp32 terms: only the fp32 du and the final rounding
    _check_within(name + " dbeta", dbeta.double(), ref["dbeta"],
                  2.0 ** -20 * du.abs().sum(dim=(0, 2, 3)) + slack + 1e-30)
    _check_within(name + " dgamma", dgamma.double(), ref["dgamma"],
                  2.0 ** -20 * (du * xh).abs().sum(dim=(0, 2, 3)) + slack * xh.abs().amax(dim=(0, 2, 3)) + 1e-30)
    N = B * H * W
    A = _ch(sc.abs())
    if training:
        S1, S2 = du.sum(dim=(0, 2, 3)), (du * xh).sum(dim=(0, 2, 3))
        # the fp32 terms du and du * (z - mean) of the sums round by 2^-22 of their magnitudes
        t1, t2 = du.abs().sum(dim=(0, 2, 3)), (du * xh).abs().sum(dim=(0, 2, 3))
        terms = A * (du.abs() + dy64.abs() * mag / 4 + _ch(S1.abs() + slack + t1 / 4) / N
                     + xh.abs() * _ch(t2 / 4) / N
                     + (z64.abs() + _ch(mean.abs())) * _ch(invstd * (S2.abs() + slack * xh.abs().amax(dim=(0, 2, 3))))
                     / N)
    else:
        terms = A * (du.abs() + dy64.abs() * mag / 4)
        assert bool((coef[1:] == 0).all())
        assert torch.equal(coef[0], (gamma.double() * save[1].double()).float())
        if act == "linear":
            # du = dy exactly, so dz = fp32(coef[0] * dy) bit for bit
            assert torch.equal(dz, coef[0] * dy), "eval dz is not coef[0] * du"
    _check_within(name + " dz", _nchw64(dz), ref["dz"], 2.0 ** -20 * terms + 1e-30, (~near).double())


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bn_train_refusals_are_errors():
    """Launches the fp16 passes cannot run are B2YError, never silent output: C not a multiple of 8, C > 2048, a pixel
    pitch that is not a multiple of 8, and no pixels"""
    import ctypes
    lib, ops = _lib()
    from b200yolo.lib import B2YError
    buf = torch.zeros(4 * 2056 * 8, dtype=torch.float16, device="cuda")
    f32 = torch.zeros(8 * 2056, dtype=torch.float32, device="cuda")
    p, fp, st = lib.ptr(buf), lib.ptr(f32), lib.stream_ptr()
    aux2 = ctypes.c_void_p(f32.data_ptr() + 4)

    def fwd(c, pitch, pixels):
        lib.call("b2y_bn_train_fwd", p, pitch, fp, fp, 4, fp, fp, EPS, MOMENTUM, fp, fp, fp, None, 0, p, pitch,
                 pixels, c, lib.ACT["leaky"], SLOPE, st)

    def red(c, pitch, pixels):
        lib.call("b2y_bn_train_bwd_reduce", p, pitch, p, pitch, fp, fp, fp, pixels, c, lib.ACT["leaky"], SLOPE,
                 lib.DT_F16, st)

    def app(c, pitch, pixels):
        lib.call("b2y_bn_train_bwd_apply", p, pitch, p, pitch, fp, fp, fp, p, pitch, pixels, c, lib.ACT["leaky"],
                 SLOPE, lib.DT_F16, fp, aux2, fp, fp, 1.0, st)

    for launch in (fwd, red, app):
        for c, pitch, pixels in ((20, 24, 4), (2056, 2056, 4), (64, 68, 4), (64, 64, 0), (64, 64, -3)):
            with pytest.raises(B2YError):
                launch(c, pitch, pixels)
    torch.cuda.synchronize()
