"""Every launch configuration of the implicit-GEMM convolution (csrc/conv_tc.cu gemm_conv_launch, kernel in
csrc/conv_tc.cuh) against fp64, at the shapes training runs: the forward, its batch statistics and the data gradient.

The host picks, per launch, the N tile (32 / 64 / 128 from the output width), the k-step width (32 / 64 / 128 bytes
from the input width), a 2-CTA weight-multicast cluster, the weight-stationary mode and one of three epilogues (TMA
store, register store, general).  Training BatchNorm statistics ride on three paths: deferred per warp on the short
epilogue when there is one N tile, flushed per chunk on the short epilogue otherwise, and the general epilogue's own.
fwd_plan / dgrad_plan below restate that choice in Python, and every case asserts the plan it was written for, so a
heuristic change that moves a case off its path fails here and the table has to be updated with it.

Each case reads its input through a channel slice of a wider buffer whose other channels (and, for the 16-channel
rounded K views of layout.py view_k, the pad channels inside the view, which meet zero weight columns) hold +-60000,
and writes into a channel slot of a sentinel-filled buffer that must come back untouched."""
import math
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

SMS = 132          # H100 SXM; the expected plans below are for this SM count
SENTINEL = -768.0  # exact in fp16, bf16 and fp32
HUGE = 60000.0     # finite in fp16; any read of these channels shows up in the result


# ---------------------------------------------------------------------------------------------------------------
# the launch plan, transcribed from gemm_conv_launch / pick_cluster / conv_max_stage_smem / enumerate_dgrad_phases
# ---------------------------------------------------------------------------------------------------------------
CONV_SMEM_LIMIT = 227 * 1024


def conv_max_stage_smem(block_n):
    return ((CONV_SMEM_LIMIT - 1024 - 1024 - 8 * 4096 - 128 * block_n * 4) // 1024) * 1024


def pick_cluster(block_n, kbytes, num_m_tiles):
    if kbytes != 128 or block_n < 128:
        return 1
    return 1 if num_m_tiles < 4 else 2


def launch_plan(M, C, nout, ntaps, sms, identity=True, out="f16", act="linear", slope=0.1, bias=False, res=False,
                stats=False, aligned=True):
    """One fp16/bf16 gemm_conv_launch over M GEMM rows, C input channels per tap and nout output channels; None where
    the host refuses it.  `aligned`: output, bias and residual 16-byte aligned with vector-multiple pitches."""
    kb_total = 2 * C
    if kb_total % 32:
        return None
    kbytes = 128 if kb_total % 128 == 0 else (64 if kb_total % 64 == 0 else 32)
    block_n = 32 if nout <= 32 else (64 if nout <= 64 else 128)
    m_tiles, n_tiles = -(-M // 128), -(-nout // block_n)
    act_ok = act in ("linear", "mish") or (act == "leaky" and 0.0 <= slope <= 1.0)
    out16 = out in ("f16", "bf16")
    full = nout % block_n == 0
    # the TMA store writes whole 16-byte pieces of a row, so it clips only widths that end on one
    clip_ok = identity and nout * (4 if out == "f32" else 2) % 16 == 0
    stats_ok = not stats or (out16 and identity and not bias and not res)
    epi_fast = ((out16 or (out == "f32" and identity)) and stats_ok and act_ok and aligned and
                (full or (clip_ok and not res)))
    epi_tma = epi_fast and identity
    cluster = pick_cluster(block_n, kbytes, m_tiles)
    a_bytes, b_bytes = 128 * kbytes, block_n * kbytes
    b_resident = (cluster == 1 and n_tiles == 1 and m_tiles > sms and
                  ntaps * (kb_total // kbytes) * b_bytes + 6 * a_bytes <= conv_max_stage_smem(block_n))
    defer_stats = stats and n_tiles == 1
    return dict(block_n=block_n, kbytes=kbytes, cluster=cluster, b_resident=b_resident, epi_fast=epi_fast,
                epi_tma=epi_tma, num_m_tiles=m_tiles, num_n_tiles=n_tiles, defer_stats=defer_stats,
                clipped=not full,
                epi="tma" if epi_tma else ("reg" if epi_fast else "general"),
                stats=None if not stats else ("general" if not epi_fast else ("deferred" if defer_stats else "chunk")))


def fwd_plan(B, H, W, C, cout, k, stride, sms, **epi):
    """conv_tc_launch (dense weights): one launch, or None if refused."""
    if k * k > 16:
        return None
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    return launch_plan(B * Ho * Wo, C, cout, k * k, sms, **epi)


def stem_plan(B, H, W, cout, k, stride, sms, **epi):
    """b2y_stem_conv_fwd_tc with in_c * k * k <= 32: one plain GEMM over the 32-column im2col workspace."""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    return launch_plan(B * Ho * Wo, 32, cout, 1, sms, **epi)


def dgrad_phases(H, W, k, stride, pad):
    """(py, px, taps, MH, MW) per output phase, in launch order."""
    out = []
    for py in range(stride):
        for px in range(stride):
            nh = sum(1 for r in range(k) if (py + pad - r) % stride == 0)
            nw = sum(1 for c in range(k) if (px + pad - c) % stride == 0)
            out.append((py, px, nh * nw, (H - py + stride - 1) // stride, (W - px + stride - 1) // stride))
    return out


def dgrad_plan(B, H, W, cin, cout, k, stride, sms, out="f16", accumulate=False, aligned=True):
    """b2y_conv2d_bwd_data: one launch per output phase (dY channels are the GEMM K, dX channels its N); None if
    refused.  An overwrite whose kernel is smaller than the stride has an untouched phase and is refused."""
    if k > 4 or stride > 4:
        return None
    plans = []
    for py, px, taps, MH, MW in dgrad_phases(H, W, k, stride, (k - 1) // 2):
        if MH <= 0 or MW <= 0:
            continue
        if taps == 0:
            if accumulate:
                continue
            return None
        p = launch_plan(B * MH * MW, cout, cin, taps, sms, identity=stride == 1, out=out, res=accumulate,
                        aligned=aligned)
        if p is None:
            return None
        plans.append(dict(p, phase=(py, px), taps=taps))
    return plans


def summary(p):
    return (p["block_n"], p["kbytes"], p["cluster"], p["b_resident"], p["epi"])


def check_plan(p, expect, sms):
    """the case's expected (block_n, kbytes, cluster, b_resident, epilogue[, statistics path]); b_resident depends
    on the SM count and is only pinned for the 132-SM part."""
    got = summary(p) + ((p["stats"],) if len(expect) > 5 else ())
    if sms != SMS:
        got, expect = got[:3] + got[4:], tuple(expect[:3]) + tuple(expect[4:])
    assert got == tuple(expect), "launch plan moved: %s, expected %s" % (got, expect)


# ---------------------------------------------------------------------------------------------------------------
# case tables
# ---------------------------------------------------------------------------------------------------------------
# cin = real input channels, ck = channels of the K view (cin rounded up to 16 as view_k does)
Fwd = namedtuple("Fwd", "B H W cin ck cout k s act slope bias res f32 expect")
FWD_CASES = {
    # more M tiles than SMs for every (block_n, kbytes) pair: the persistent loop over many tiles per CTA
    "c16-32_k3_104": Fwd(8, 104, 104, 16, 16, 32, 3, 1, "leaky", 0.2, True, False, False, (32, 32, 1, True, "tma")),
    "c24-32_k3_104": Fwd(8, 104, 104, 24, 32, 32, 3, 1, "leaky", 0.125, True, False, False, (32, 64, 1, True, "tma")),
    "c64-32_k1_208": Fwd(8, 208, 208, 64, 64, 32, 1, 1, "leaky", 0.1, True, False, False, (32, 128, 1, True, "tma")),
    "c16-48_k1_104": Fwd(8, 104, 104, 16, 16, 48, 1, 1, "relu6", 0.1, True, False, False,
                         (64, 32, 1, True, "general")),
    # yolov3's second layer at 416 px, batch 8
    "c32-64_k3s2_416": Fwd(8, 416, 416, 32, 32, 64, 3, 2, "leaky", 0.1, True, False, False, (64, 64, 1, True, "tma")),
    "c128-64_k1_104_res": Fwd(8, 104, 104, 128, 128, 64, 1, 1, "leaky", 0.2, True, True, False,
                              (64, 128, 1, True, "tma")),
    "c40-120_k1_51x53": Fwd(8, 51, 53, 40, 48, 120, 1, 1, "h_swish", 0.1, True, False, False,
                            (128, 32, 1, True, "general")),
    "c32-128_k3_104": Fwd(8, 104, 104, 32, 32, 128, 3, 1, "mish", 0.1, True, False, False,
                          (128, 64, 1, True, "tma")),
    "c64-128_k3s2_208": Fwd(8, 208, 208, 64, 64, 128, 3, 2, "leaky", 0.25, True, False, False,
                            (128, 128, 2, False, "tma")),
    # one or two M tiles: no cluster
    "c64-128_k3_16": Fwd(1, 16, 16, 64, 64, 128, 3, 1, "leaky", 0.2, True, False, False, (128, 128, 1, False, "tma")),
    # fp32 heads in a 256-channel buffer; 169 M tiles under cluster 2 leave the last cluster's second tile without
    # rows.  255 columns end inside a 16-byte piece, which the TMA store would write whole (column 255): the general
    # epilogue stores them.  252 columns end on one: the TMA store clips the last tile.
    "head_c256-255_k1_52": Fwd(8, 52, 52, 256, 256, 255, 1, 1, "linear", 0.1, True, False, True,
                               (128, 128, 2, False, "general")),
    "head_c256-252_k1_52": Fwd(8, 52, 52, 256, 256, 252, 1, 1, "linear", 0.1, True, False, True,
                               (128, 128, 2, False, "tma")),
    # 40 fp16 channels = 80 bytes: clipped on a 16-byte but not a 32-byte boundary
    "c32-40_k1_26": Fwd(8, 26, 26, 32, 32, 40, 1, 1, "leaky", 0.2, True, False, False, (64, 64, 1, False, "tma")),
    # MobileNet widths: N 960 (clipped last tile), K 960, K 80 / N 208 with a residual, K 200 -> 208 / N 80
    "c160-960_k1_13": Fwd(8, 13, 13, 160, 160, 960, 1, 1, "linear", 0.1, True, False, False,
                          (128, 64, 1, False, "tma")),
    "c960-160_k1_13": Fwd(8, 13, 13, 960, 960, 160, 1, 1, "relu6", 0.1, True, False, False,
                          (128, 128, 2, False, "general")),
    "c80-208_k1_26_res": Fwd(8, 26, 26, 80, 80, 208, 1, 1, "linear", 0.1, True, True, False,
                             (128, 32, 1, False, "general")),
    "c200-80_k3s2_27": Fwd(4, 27, 27, 200, 208, 80, 3, 2, "h_swish", 0.1, True, False, False,
                           (128, 32, 1, False, "general")),
}

# statistics: linear, no residual; a bias sends the launch to the general epilogue (its sums stay pre-bias)
Stat = namedtuple("Stat", "B H W cin ck cout k s bias offset expect")
STATS_CASES = {
    "deferred_c32-64_k3s2_416": Stat(8, 416, 416, 32, 32, 64, 3, 2, False, 0.0,
                                     (64, 64, 1, True, "tma", "deferred")),
    # channel means of 8 sigma: the fp32 E[z^2] - E[z]^2 of bn_train_fwd cancels 6 of its 24 bits
    "deferred_c128-64_k1_104_mean8sigma": Stat(8, 104, 104, 128, 128, 64, 1, 1, False, 8.0,
                                               (64, 128, 1, True, "tma", "deferred")),
    # yolov3's downsampling layers at 416 px, batch 8: 169 / 43 / 11 M tiles, odd, under cluster 2
    "chunk_c128-256_k3s2_104": Stat(8, 104, 104, 128, 128, 256, 3, 2, False, 0.0,
                                    (128, 128, 2, False, "tma", "chunk")),
    "chunk_c256-512_k3s2_52": Stat(8, 52, 52, 256, 256, 512, 3, 2, False, 0.0,
                                   (128, 128, 2, False, "tma", "chunk")),
    "chunk_c512-1024_k3s2_26": Stat(8, 26, 26, 512, 512, 1024, 3, 2, False, 0.0,
                                    (128, 128, 2, False, "tma", "chunk")),
    "chunk_c160-960_k1_13": Stat(8, 13, 13, 160, 160, 960, 1, 1, False, 0.0, (128, 64, 1, False, "tma", "chunk")),
    "general_c64-128_k3_104_bias": Stat(8, 104, 104, 64, 64, 128, 3, 1, True, 0.0,
                                        (128, 128, 2, False, "general", "general")),
    "general_c80-208_k1_52_bias": Stat(8, 52, 52, 80, 80, 208, 1, 1, True, 0.0,
                                       (128, 32, 1, False, "general", "general")),
    # clipped N tiles on the short path
    "deferred_c40-80_k1_52": Stat(8, 52, 52, 40, 48, 80, 1, 1, False, 0.0, (128, 32, 1, True, "tma", "deferred")),
    "chunk_c80-208_k1_52": Stat(8, 52, 52, 80, 80, 208, 1, 1, False, 0.0, (128, 32, 1, False, "tma", "chunk")),
}

# the full-resolution stem: 3 -> 32, 3x3, 416 px, batch 8 (1.4M pixels, the largest reduction in training)
STEM = dict(B=8, H=416, W=416, cin=3, cout=32, k=3, s=1, expect=(32, 64, 1, True, "tma", "deferred"))

# dX (in_c channels, the GEMM N) from dY (out_c channels, the GEMM K); `expect` holds for every phase
Dgrad = namedtuple("Dgrad", "B H W cin cout k s opd outd inv acc expect")
DGRAD_CASES = {
    # yolov3's training size: 64 -> 128, 3x3, stride 2, from 208 px at batch 8; fp16 dY, bf16 dX accumulated in place
    "c64-128_k3s2_208_acc_bf16": Dgrad(8, 208, 208, 64, 128, 3, 2, "f16", "bf16", True, True,
                                       (64, 128, 1, True, "reg")),
    "c128-256_k3s1_27x25": Dgrad(4, 27, 25, 128, 256, 3, 1, "f16", "f16", False, False, (128, 128, 2, False, "tma")),
    "c80-160_k3s2_33x31_acc": Dgrad(2, 33, 31, 80, 160, 3, 2, "bf16", "bf16", False, True,
                                    (128, 64, 1, False, "general")),
    "c48-96_k3s2_40": Dgrad(2, 40, 40, 48, 96, 3, 2, "f16", "f16", True, False, (64, 64, 1, False, "general")),
    "c208-80_k1s1_26_acc": Dgrad(2, 26, 26, 208, 80, 1, 1, "f16", "bf16", True, True,
                                 (128, 32, 1, False, "general")),
    # kernel smaller than the stride: only phase (0, 0) has taps; the accumulate form leaves the others as they were
    "c64-128_k1s2_20x21_acc": Dgrad(2, 20, 21, 64, 128, 1, 2, "f16", "f16", False, True, (64, 128, 1, False, "reg")),
    "c64-128_k3s2_27x29": Dgrad(2, 27, 29, 64, 128, 3, 2, "bf16", "f16", False, False, (64, 128, 1, False, "reg")),
    "c128-64_k3s2_30_acc": Dgrad(4, 30, 30, 128, 64, 3, 2, "f16", "f16", True, True, (128, 128, 2, False, "reg")),
    "c64-32_k3s1_24_acc_bf16": Dgrad(2, 24, 24, 64, 32, 3, 1, "bf16", "bf16", True, True,
                                     (64, 64, 1, False, "tma")),
    "c48-64_k3s1_20": Dgrad(2, 20, 20, 48, 64, 3, 1, "f16", "f16", False, False, (64, 128, 1, False, "tma")),
}


def _fwd_case_plan(c, sms, aligned=True):
    return fwd_plan(c.B, c.H, c.W, c.ck, c.cout, c.k, c.s, sms, out="f32" if c.f32 else "f16", act=c.act,
                    slope=c.slope, bias=c.bias, res=c.res, aligned=aligned)


def _stats_case_plan(c, sms, aligned=True):
    return fwd_plan(c.B, c.H, c.W, c.ck, c.cout, c.k, c.s, sms, bias=c.bias, stats=True, aligned=aligned)


def _stem_plan(sms):
    return stem_plan(STEM["B"], STEM["H"], STEM["W"], STEM["cout"], STEM["k"], STEM["s"], sms, stats=True)


def _dgrad_case_plan(c, sms, aligned=True):
    return dgrad_plan(c.B, c.H, c.W, c.cin, c.cout, c.k, c.s, sms, out=c.outd, accumulate=c.acc, aligned=aligned)


def test_case_table_covers_every_launch_path():
    """Runs without a GPU: every case lands on the plan it names, and together they reach every launch variant."""
    plans = []
    for c in FWD_CASES.values():
        p = _fwd_case_plan(c, SMS)
        check_plan(p, c.expect, SMS)
        plans.append(p)
    for c in STATS_CASES.values():
        p = _stats_case_plan(c, SMS)
        check_plan(p, c.expect, SMS)
        plans.append(p)
    p = _stem_plan(SMS)
    check_plan(p, STEM["expect"], SMS)
    plans.append(p)
    for c in DGRAD_CASES.values():
        ph = _dgrad_case_plan(c, SMS)
        assert ph
        for p in ph:
            check_plan(p, c.expect, SMS)
        plans += ph
    pairs = {(bn, kb) for bn in (32, 64, 128) for kb in (32, 64, 128)}
    assert {(p["block_n"], p["kbytes"]) for p in plans if p["cluster"] == 1} == pairs
    assert any(p["cluster"] == 2 for p in plans)
    # training scale: every tile shape with more M tiles than SMs, in the forward
    fwd = [_fwd_case_plan(c, SMS) for c in FWD_CASES.values()]
    assert {(p["block_n"], p["kbytes"]) for p in fwd if p["num_m_tiles"] > SMS} == pairs
    assert {p["b_resident"] for p in plans} == {True, False}
    assert {p["epi"] for p in plans} == {"tma", "reg", "general"}
    assert {p["stats"] for p in plans} - {None} == {"deferred", "chunk", "general"}
    assert any(p["cluster"] == 2 and p["num_m_tiles"] % 2 == 1 for p in plans)
    assert any(p["cluster"] == 2 and p["num_m_tiles"] % 2 == 1 and p["stats"] for p in plans)
    # the register-store epilogue needs whole N tiles; the other two clip the last one
    assert {p["epi"] for p in plans if p["clipped"]} == {"tma", "general"}
    assert any(p["clipped"] and p["stats"] == "deferred" for p in plans)
    assert any(p["clipped"] and p["stats"] == "chunk" for p in plans)
    assert any(p["clipped"] and p["stats"] == "general" for p in plans)
    # the data gradient's register stores with both residual formats (in-place fp16 and bf16 accumulation)
    assert {c.outd for c in DGRAD_CASES.values() if c.acc and c.expect[4] == "reg"} == {"f16", "bf16"}
    assert {(c.opd, c.outd) for c in DGRAD_CASES.values()} == {(a, b) for a in ("f16", "bf16") for b in ("f16", "bf16")}
    # the refusals exercised by test_conv_refusals_are_errors
    assert dgrad_plan(2, 20, 21, 64, 128, 1, 2, SMS, accumulate=False) is None
    assert dgrad_plan(2, 20, 20, 64, 64, 5, 1, SMS) is None
    assert fwd_plan(2, 20, 20, 64, 64, 5, 1, SMS) is None
    assert fwd_plan(2, 20, 20, 24, 64, 3, 1, SMS) is None
    assert dgrad_plan(2, 20, 20, 64, 24, 3, 1, SMS) is None


# ---------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------
def _ops():
    from b200yolo import ops
    return ops


def _seed(name):
    return zlib.crc32(name.encode()) % 10007


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _al16(t):
    return t.data_ptr() % 16 == 0


def _huge_buffer(g, shape, dtype):
    """+-HUGE everywhere: channels a launch must never read"""
    sign = torch.randint(0, 2, shape, generator=g, device="cuda", dtype=torch.int8)
    return (sign.to(dtype) * 2 - 1) * HUGE


def _input_view(g, B, H, W, cin, ck, dtype=torch.float16):
    """x as channels [8, 8 + ck) of a wider NHWC buffer: the real channels are [0, cin) of the view; the view's pad
    channels (view_k) and everything outside it hold +-HUGE.  Returns (view, fp64 NCHW of the real channels)."""
    buf = _huge_buffer(g, (B, H, W, 8 + ck + 8), dtype)
    buf[..., 8:8 + cin] = torch.randn(B, H, W, cin, generator=g, device="cuda").to(dtype)
    xv = buf[..., 8:8 + ck]
    return xv, xv[..., :cin].permute(0, 3, 1, 2).double()


def _packed_weights(g, cout, cin, ck, k):
    """fp16 OIHW weights and their [O][k][k][ck] pack with zero columns at the view's pad channels"""
    w = (torch.randn(cout, cin, k, k, generator=g, device="cuda") / math.sqrt(cin * k * k)).half()
    wp = torch.zeros(cout, k, k, ck, dtype=torch.float16, device="cuda")
    wp[..., :cin] = w.permute(0, 2, 3, 1)
    return w, wp


def _output_slot(B, Ho, Wo, cout, dtype, lead, trail):
    """(buffer, view): channels [lead, lead + cout) of a sentinel-filled buffer"""
    buf = torch.full((B, Ho, Wo, lead + cout + trail), SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[..., lead:lead + cout]


def _assert_slot_only(buf, lead, n):
    s = torch.full((), SENTINEL, dtype=buf.dtype, device=buf.device)
    assert bool((buf[..., :lead] == s).all()) and bool((buf[..., lead + n:] == s).all()), \
        "wrote outside the channel slot"


def _aligned(out, res=None, out_vec=8):
    pitch = out.stride(2)
    ok = _al16(out) and pitch % out_vec == 0
    if res is not None:
        ok = ok and _al16(res) and res.stride(2) % 8 == 0
    return ok


def _act64(y, act, slope):
    if act == "leaky":
        return torch.where(y > 0, y, y * slope)
    if act == "relu6":
        return y.clamp(0.0, 6.0)
    if act == "h_swish":
        return y * (y + 3.0).clamp(0.0, 6.0) / 6.0
    if act == "mish":
        return y * torch.tanh(F.softplus(y))
    return y


def _nchw64(t):
    return t.permute(0, 3, 1, 2).double()


def _print_plan(tag, p, **numbers):
    keys = ("block_n", "kbytes", "cluster", "b_resident", "epi_fast", "epi_tma", "num_m_tiles", "num_n_tiles",
            "defer_stats")
    extra = " ".join("%s %.3g" % kv for kv in numbers.items())
    print("\n%s: %s %s" % (tag, " ".join("%s=%s" % (k, int(p[k]) if isinstance(p[k], bool) else p[k]) for k in keys),
                           extra))


# ---------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FWD_CASES))
def test_conv_forward_plan_against_fp64(name):
    c = FWD_CASES[name]
    ops = _ops()
    sms = _sms()
    g = torch.Generator(device="cuda").manual_seed(_seed(name))
    pad = (c.k - 1) // 2
    Ho, Wo = (c.H + 2 * pad - c.k) // c.s + 1, (c.W + 2 * pad - c.k) // c.s + 1
    xv, x64 = _input_view(g, c.B, c.H, c.W, c.cin, c.ck)
    w, wp = _packed_weights(g, c.cout, c.cin, c.ck, c.k)
    bias = torch.randn(c.cout, generator=g, device="cuda") * 0.5 if c.bias else None
    res = torch.randn(c.B, Ho, Wo, c.cout, generator=g, device="cuda").half() if c.res else None
    if c.f32:       # the head's raw buffer is 256 channels wide; the columns past the head keep their sentinel
        lead, trail, odt = 0, 256 - c.cout, torch.float32
    else:
        lead, trail, odt = 8, 8, torch.float16
    obuf, ov = _output_slot(c.B, Ho, Wo, c.cout, odt, lead, trail)
    aligned = _aligned(ov, res, 4 if c.f32 else 8)
    assert aligned
    p = _fwd_case_plan(c, sms, aligned)
    check_plan(p, c.expect, sms)

    ops.conv2d(xv, wp, bias, c.k, c.s, pad, act=c.act, slope=c.slope, residual=res, out=ov)
    ref = F.conv2d(x64, w.double(), bias.double() if bias is not None else None, stride=c.s, padding=pad)
    ref = _act64(ref, c.act, c.slope)
    if res is not None:
        ref = ref + _nchw64(res)
    err = (_nchw64(ov) - ref).abs().max().item()
    rms = ref.pow(2).mean().sqrt().item()
    _print_plan(name, p, err=err, rms=rms, err_over_rms=err / rms)
    _assert_slot_only(obuf, lead, c.cout)
    # fp16 store: half an ulp is 2^-11 of |y|, and |y| stays below 8 rms at these sizes; fp32: accumulation order only
    tol = 2e-5 if c.f32 else 4e-3
    assert err <= tol * max(rms, 1.0), "max err %g rms %g" % (err, rms)


# ---------------------------------------------------------------------------------------------------------------
# batch statistics
# ---------------------------------------------------------------------------------------------------------------
def _check_stats(tag, p, launch, z64, has_bias):
    """launch(s1, s2) adds the batch sums of one convolution into s1, s2 and returns the fp16 z it wrote.
    Against the fp64 sums of z64 (NCHW): fresh sums, accumulation into pre-filled ones, bit-identical repeats (the
    per-stream fp64 accumulator is cleared between launches), and bn_train_fwd's mean / invstd / running variance."""
    ops = _ops()
    cout = z64.shape[1]
    M = z64.numel() // cout
    dev = "cuda"
    ref1 = z64.sum(dim=(0, 2, 3))
    ref2 = z64.square().sum(dim=(0, 2, 3))
    # fp32 partial sums over at most a few thousand rows, added in fp64: 1e-5 of the sum of |terms| bounds them
    tol1 = 1e-5 * z64.abs().sum(dim=(0, 2, 3))
    tol2 = 1e-5 * ref2

    s1 = torch.zeros(cout, device=dev)
    s2 = torch.zeros(cout, device=dev)
    z = launch(s1, s2)
    e1 = ((s1.double() - ref1).abs() / tol1).max().item()
    e2 = ((s2.double() - ref2).abs() / tol2).max().item()

    g = torch.Generator(device=dev).manual_seed(5)
    base1 = torch.randn(cout, generator=g, device=dev) * ref1.abs().max().float()
    base2 = torch.rand(cout, generator=g, device=dev) * ref2.max().float()
    a1, a2 = base1.clone(), base2.clone()
    launch(a1, a2)
    b1, b2 = base1.clone(), base2.clone()
    launch(b1, b2)
    want1, want2 = base1.double() + ref1, base2.double() + ref2
    # one more fp32 rounding of the pre-filled value
    ea1 = ((a1.double() - want1).abs() / (tol1 + 2.0 ** -23 * want1.abs())).max().item()
    ea2 = ((a2.double() - want2).abs() / (tol2 + 2.0 ** -23 * want2.abs())).max().item()

    chain = {}
    if not has_bias:
        gamma = torch.rand(cout, generator=g, device=dev) + 0.5
        beta = torch.randn(cout, generator=g, device=dev) * 0.2
        rm = torch.randn(cout, generator=g, device=dev) * 0.1
        rv = torch.rand(cout, generator=g, device=dev) + 0.5
        rm0, rv0 = rm.double(), rv.double()
        _, save = ops.bn_train_fwd(z, s1, s2, gamma, beta, 1e-5, 0.1, rm, rv, "linear")
        mean = z64.mean(dim=(0, 2, 3))
        var = (z64 - mean.view(1, -1, 1, 1)).square().mean(dim=(0, 2, 3))     # two-pass
        invstd = 1.0 / torch.sqrt(var + 1e-5)
        rv_ref = 0.9 * rv0 + 0.1 * var * (M / (M - 1))
        rm_ref = 0.9 * rm0 + 0.1 * mean
        # the mean relative to the channel's scale (a zero-mean channel has no relative error to speak of)
        chain = dict(
            mean=((save[0].double() - mean).abs() / (mean.abs() + var.sqrt())).max().item(),
            invstd=((save[1].double() - invstd).abs() / invstd).max().item(),
            running_var=((rv.double() - rv_ref).abs() / rv_ref).max().item(),
            running_mean=((rm.double() - rm_ref).abs() / (rm_ref.abs() + 0.1 * var.sqrt())).max().item(),
            mean_over_sigma=(mean.abs() / var.sqrt()).median().item())
    _print_plan(tag, p, sum_err=e1, sq_err=e2, acc_sum_err=ea1, acc_sq_err=ea2, **chain)
    assert e1 <= 1.0 and e2 <= 1.0, "batch sums off: %g %g (units of the tolerance)" % (e1, e2)
    assert ea1 <= 1.0 and ea2 <= 1.0, "sums do not accumulate into the pre-filled buffers: %g %g" % (ea1, ea2)
    assert torch.equal(a1, b1) and torch.equal(a2, b2), "a repeated launch gives different sums"
    if chain:
        assert chain["mean"] <= 1e-4 and chain["invstd"] <= 1e-4, chain
        assert chain["running_var"] <= 1e-4 and chain["running_mean"] <= 1e-4, chain


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STATS_CASES))
def test_conv_batch_statistics_against_fp64(name):
    c = STATS_CASES[name]
    ops = _ops()
    sms = _sms()
    g = torch.Generator(device="cuda").manual_seed(_seed(name) + 7)
    pad = (c.k - 1) // 2
    Ho, Wo = (c.H + 2 * pad - c.k) // c.s + 1, (c.W + 2 * pad - c.k) // c.s + 1
    xv, x64 = _input_view(g, c.B, c.H, c.W, c.cin, c.ck)
    w, wp = _packed_weights(g, c.cout, c.cin, c.ck, c.k)
    if c.offset:
        # input channel 0 is 1 everywhere (1x1: no border), and its weight gives each output channel a mean of
        # `offset` times its standard deviation
        assert c.k == 1
        xv[..., 0] = 1.0
        x64 = xv[..., :c.cin].permute(0, 3, 1, 2).double()
        sigma = w[:, 1:].float().pow(2).sum(dim=(1, 2, 3)).sqrt()
        w[:, 0, 0, 0] = (c.offset * sigma).half()
        wp[:, 0, 0, 0] = w[:, 0, 0, 0]
    bias = torch.randn(c.cout, generator=g, device="cuda") * 0.5 if c.bias else None
    obuf, ov = _output_slot(c.B, Ho, Wo, c.cout, torch.float16, 8, 8)
    aligned = _aligned(ov)
    assert aligned
    p = _stats_case_plan(c, sms, aligned)
    check_plan(p, c.expect, sms)
    z64 = F.conv2d(x64, w.double(), None, stride=c.s, padding=pad)

    def launch(s1, s2):
        ops.conv2d(xv, wp, bias, c.k, c.s, pad, out=ov, stats=(s1, s2))
        return ov

    _check_stats(name, p, launch, z64, c.bias)
    ref = z64 + bias.double().view(1, -1, 1, 1) if c.bias else z64
    err = (_nchw64(ov) - ref).abs().max().item()
    rms = ref.pow(2).mean().sqrt().item()
    print("output err %.3g rms %.3g" % (err, rms))
    _assert_slot_only(obuf, 8, c.cout)
    assert err <= 4e-3 * max(rms, 1.0), (err, rms)


@pytest.mark.gpu
def test_stem_batch_statistics_full_resolution():
    """b2y_stem_conv_fwd_tc with statistics: 3 -> 32, 3x3, 416 px, batch 8 (1.4M pixels)."""
    ops = _ops()
    sms = _sms()
    s = STEM
    g = torch.Generator(device="cuda").manual_seed(17)
    x = torch.rand(s["B"], s["cin"], s["H"], s["W"], generator=g, device="cuda")
    w = torch.randn(s["cout"], s["cin"], s["k"], s["k"], generator=g, device="cuda") / 5
    ws = ops.pack_stem_weights(w)
    p = _stem_plan(sms)
    check_plan(p, s["expect"], sms)
    obuf, ov = _output_slot(s["B"], s["H"], s["W"], s["cout"], torch.float16, 8, 8)
    workspace = []

    def launch(s1, s2):
        _, wsp = ops.stem_conv_tc(x, ws, None, s["cin"], s["k"], s["s"], s["k"] // 2, out=ov, stats=(s1, s2),
                                  workspace=workspace[0] if workspace else None)
        workspace[:] = [wsp]
        return ov

    # the pack rounds the image and the weights to fp16
    z64 = F.conv2d(x.half().double(), w.half().double(), None, stride=s["s"], padding=s["k"] // 2)
    _check_stats("stem_c3-32_k3_416", p, launch, z64, False)
    err = (_nchw64(ov) - z64).abs().max().item()
    rms = z64.pow(2).mean().sqrt().item()
    _assert_slot_only(obuf, 8, s["cout"])
    assert err <= 4e-3 * max(rms, 1.0), (err, rms)


# ---------------------------------------------------------------------------------------------------------------
# data gradient
# ---------------------------------------------------------------------------------------------------------------
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
HALF_ULP = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DGRAD_CASES))
def test_conv_data_gradient_plan_against_fp64(name):
    """dX written into (or accumulated into) channels [16, 16 + cin) of a wider sentinel-filled gradient buffer, as
    the training engine does for a route source, from dY read as a channel slice of a wider buffer."""
    c = DGRAD_CASES[name]
    ops = _ops()
    sms = _sms()
    g = torch.Generator(device="cuda").manual_seed(_seed(name) + 3)
    pad = (c.k - 1) // 2
    Ho, Wo = (c.H + 2 * pad - c.k) // c.s + 1, (c.W + 2 * pad - c.k) // c.s + 1
    opd, outd = DT[c.opd], DT[c.outd]
    w = torch.randn(c.cout, c.cin, c.k, c.k, generator=g, device="cuda") / math.sqrt(c.cout * c.k * c.k / c.s ** 2)
    wt = ops.pack_dgrad_weights(w, c.s, pad, (c.H, c.W), dtype=opd)
    dyb = _huge_buffer(g, (c.B, Ho, Wo, 8 + c.cout + 8), opd)
    dyb[..., 8:8 + c.cout] = torch.randn(c.B, Ho, Wo, c.cout, generator=g, device="cuda").to(opd)
    dyv = dyb[..., 8:8 + c.cout]
    gbuf, dxv = _output_slot(c.B, c.H, c.W, c.cin, outd, 16, 8)
    if c.acc:
        dxv.copy_(torch.randn(c.B, c.H, c.W, c.cin, generator=g, device="cuda").to(outd))
    base = _nchw64(dxv) if c.acc else None
    aligned = _aligned(dxv, dxv if c.acc else None)
    assert aligned
    phases = _dgrad_case_plan(c, sms, aligned)
    for p in phases:
        check_plan(p, c.expect, sms)
    inv = torch.tensor([0.3], device="cuda") if c.inv else None

    ops.conv2d_bwd_data(dyv, wt, (c.B, c.H, c.W, c.cin), c.k, c.s, pad, out=dxv, accumulate=c.acc, inv_scale=inv)
    ref = torch.nn.grad.conv2d_input((c.B, c.cin, c.H, c.W), w.to(opd).double(), _nchw64(dyv), stride=c.s,
                                     padding=pad)
    if inv is not None:
        ref = ref * inv.double()
    if base is not None:
        ref = ref + base
    err = (_nchw64(dxv) - ref).abs().max().item()
    rms = ref.pow(2).mean().sqrt().item()
    amax = ref.abs().max().item()
    for p in phases:
        _print_plan("%s phase %s taps %d" % (name, p["phase"], p["taps"]), p)
    print("err %.3g rms %.3g err/rms %.3g" % (err, rms, err / rms))
    _assert_slot_only(gbuf, 16, c.cin)
    # one rounding to the dX format (half an ulp of |dX|) plus fp32 accumulation order
    assert err <= HALF_ULP[c.outd] * amax + 1e-3 * rms, "max err %g rms %g max|dx| %g" % (err, rms, amax)


@pytest.mark.gpu
def test_conv_refusals_are_errors():
    """Launches the kernel cannot run are B2YError, never silent output."""
    from b200yolo.lib import B2YError
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(2)
    dev = "cuda"
    # overwrite with a kernel smaller than the stride: phases (0, 1), (1, 0), (1, 1) have no taps and would need a
    # zero fill (their accumulate form is test_conv_data_gradient_plan_against_fp64[c64-128_k1s2_20x21_acc])
    w = torch.randn(128, 64, 1, 1, generator=g, device=dev)
    wt = ops.pack_dgrad_weights(w, 2, 0, (20, 21))
    dy = torch.randn(2, 10, 11, 128, generator=g, device=dev).half()
    with pytest.raises(B2YError):
        ops.conv2d_bwd_data(dy, wt, (2, 20, 21, 64), 1, 2, 0)
    # ksize^2 > 16
    w5 = torch.randn(64, 64, 5, 5, generator=g, device=dev)
    with pytest.raises(B2YError):
        ops.pack_dgrad_weights(w5, 1, 2, (20, 20))
    dy5 = torch.randn(2, 20, 20, 64, generator=g, device=dev).half()
    with pytest.raises(B2YError):
        ops.conv2d_bwd_data(dy5, torch.zeros(64 * 64 * 25, dtype=torch.float16, device=dev), (2, 20, 20, 64), 5, 1, 2)
    x5 = torch.randn(2, 20, 20, 64, generator=g, device=dev).half()
    with pytest.raises(B2YError):
        ops.conv2d(x5, torch.zeros(64, 5, 5, 64, dtype=torch.float16, device=dev), None, 5, 1, 2)
    # K bytes not a multiple of 32: 24 channels without their view_k padding
    x24 = torch.randn(2, 20, 20, 24, generator=g, device=dev).half()
    with pytest.raises(B2YError):
        ops.conv2d(x24, torch.zeros(64, 3, 3, 24, dtype=torch.float16, device=dev), None, 3, 1, 1)
    dy24 = torch.randn(2, 20, 20, 24, generator=g, device=dev).half()
    wt24 = ops.pack_dgrad_weights(torch.randn(24, 64, 3, 3, generator=g, device=dev), 1, 1, (20, 20))
    with pytest.raises(B2YError):
        ops.conv2d_bwd_data(dy24, wt24, (2, 20, 20, 64), 3, 1, 1)
    torch.cuda.synchronize()
