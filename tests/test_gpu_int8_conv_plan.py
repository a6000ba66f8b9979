"""Every launch configuration of the INT8 implicit-GEMM convolution (CONV_KIND_I8 through csrc/conv_tc.cu
gemm_conv_launch, kernel and epilogues in csrc/conv_tc.cuh), the shortcut folded into its epilogue, and the int8 graph's
other kernels, code for code against exact integer arithmetic.

The reference simulates int8 in fp32 on power-of-two grids, so the oracle below is exact where the reference is exact
and rounds, in fp32, exactly where the reference rounds, one torch op per rounding:
    acc = the conv of the integer codes in fp64 (exact below 2^53)
    a   = fp32(acc)                                  the kernel's (float)(int)acc
    v   = fp32(fp32(a * acc_scale) + bias)           one rounding fewer when acc_scale is a power of two
    v   = act(v)                                     leaky: fp32(v * fp32(slope))
    t   = v * (1 / out_scale)                        exact
    q   = clamp(sign(t) * floor(fp32(|t| + 0.5)))    the fp32 add is the reference's too (0.49999997 + 0.5 = 1)
Heads write q * out_scale in fp32, or v itself when they do not requantise.  Every comparison is torch.equal.

int8_launch_plan restates the host's choice of N tile, k-step width, cluster, weight-stationary mode and epilogue
(int8 TMA store, fp32 TMA store with or without fake-quant, general) and of the shortcut branch; every case asserts the
plan it was written for, so a change of those rules moves a case off its path and fails here.  Each case reads through a
channel slice of a wider buffer whose other channels (and the pad channels of a K view) hold +-127 / -128 codes that meet
zero weight columns, and writes into a slot of a sentinel-filled buffer.  The pixel-pair layouts of the narrow 3x3 layers
read a dense tensor (that is what the pair view needs); their outputs sit between sentinel margins instead."""
import ctypes as C
import math
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from helpers import orc

SMS = 132               # H100 SXM; the expected plans below are for this SM count
LEAD, TRAIL = 32, 16    # channels around an int8 slot (16-byte aligned, pitch a multiple of 16)
SENT8 = -99             # int8 sentinel
SENT32 = -768.0         # fp32 sentinel
OUT_SCALE = 2.0 ** -9   # activation scale of the conv cases; acc_scale = out_scale / 2^r
# h_swish(v) = v * (v + 3) / 6 >= -0.375 reaches the lowest code only at scales <= 2^-9, where none of its exact products
# lands on a rounding tie; at 2^-8 some do on both sides of zero (v = -0.1875 -> -22.5, 0.1875 -> 25.5, ...)
OUT_SCALE_HSWISH = 2.0 ** -8


# ---------------------------------------------------------------------------------------------------------------
# the launch plan, transcribed from gemm_conv_launch / conv_tc_launch with esize = 1
# ---------------------------------------------------------------------------------------------------------------
CONV_SMEM_LIMIT = 227 * 1024


def conv_max_stage_smem(block_n):
    return ((CONV_SMEM_LIMIT - 1024 - 1024 - 8 * 4096 - 128 * block_n * 4) // 1024) * 1024


def pick_cluster(block_n, kbytes, num_m_tiles):
    if kbytes != 128 or block_n < 128:
        return 1
    return 1 if num_m_tiles < 4 else 2


def _pow2(v):
    return v > 0 and math.frexp(v)[0] == 0.5


def int8_geometry(B, H, W, ck, cout, k, s, layout, dense_input=True):
    """(M, C, nout, ntaps) of the one gemm_conv_launch of an int8 conv over a ck-channel view, None where
    conv_tc_launch refuses it.  's2': B2Y_WLAYOUT_S2_PAIRS (3 x 2 taps over pixel pairs, stride 2 x 1); 's1':
    ops.s1_pair_weights over qengine._pairs views ([B,H,W/2,2C] in, [B,H,W/2,2*cout] out, 3x3 stride 1)."""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    if layout == "s2":
        if k != 3 or s != 2 or W % 2 or not dense_input or ck % 32:
            return None
        return B * Ho * Wo, 2 * ck, cout, 6
    if layout == "s1":
        assert k == 3 and s == 1 and W % 2 == 0 and dense_input
        return B * H * (W // 2), 2 * ck, 2 * cout, 9
    if k * k > 16:
        return None
    return B * Ho * Wo, ck, cout, k * k


def int8_launch_plan(M, C, nout, ntaps, sms, out="i8", act="leaky", slope=0.1, acc_pow2=True, requant=True,
                     q_lo=-128, q_hi=127, aligned=True, qres=None):
    """One CONV_KIND_I8 gemm_conv_launch; None where the host refuses it.  `aligned`: output and bias 16-byte aligned
    with a vector-multiple pitch.  `qres`: the folded shortcut, dict(out_scale, a_in, sx, sa, ssum, lo, hi, clamp,
    aligned) with aligned = addend 16-byte aligned with a pitch that is a multiple of 16."""
    if C % 32:
        return None
    kbytes = 128 if C % 128 == 0 else (64 if C % 64 == 0 else 32)
    block_n = 32 if nout <= 32 else (64 if nout <= 64 else 128)
    m_tiles, n_tiles = -(-M // 128), -(-nout // block_n)
    full = nout % block_n == 0
    int_bounds = q_lo == int(q_lo) and q_hi == int(q_hi)
    if out == "i8":
        fast = ((act == "linear" or (act == "leaky" and 0.0 <= slope <= 1.0)) and acc_pow2 and full and aligned and
                q_lo >= -128 and q_hi <= 127 and int_bounds)
        epi = "i8-tma"
    else:       # fp32 rows of the YOLO heads: the TMA store clips the last tile where the width ends on 16 bytes
        clip_ok = nout * 4 % 16 == 0
        fast = (act == "linear" and acc_pow2 and (full or clip_ok) and aligned and
                (not requant or (q_lo >= -4194304 and q_hi <= 4194303 and int_bounds)))
        epi = "f32-tma-fq" if requant else "f32-tma-linear"
    branch = None
    if qres is not None:
        r = qres
        if (not fast or out != "i8" or not r["aligned"] or
                not all(_pow2(r[n]) for n in ("out_scale", "a_in", "sx", "sa", "ssum"))):
            return None
        cx, ca = r["out_scale"] / r["ssum"], r["a_in"] / r["ssum"]
        simple = (not r["clamp"] and r["out_scale"] >= r["sx"] and r["a_in"] >= r["sa"] and
                  1.0 / 4096 <= cx <= 4096 and 1.0 / 4096 <= ca <= 4096 and r["lo"] >= -128 and r["hi"] <= 127)
        branch = "clamp" if r["clamp"] else ("simple" if simple else "rounded")
    cluster = pick_cluster(block_n, kbytes, m_tiles)
    a_bytes, b_bytes = 128 * kbytes, block_n * kbytes
    b_resident = (cluster == 1 and n_tiles == 1 and m_tiles > sms and
                  ntaps * (C // kbytes) * b_bytes + 6 * a_bytes <= conv_max_stage_smem(block_n))
    return dict(block_n=block_n, kbytes=kbytes, cluster=cluster, b_resident=b_resident, epi=epi if fast else "general",
                num_m_tiles=m_tiles, num_n_tiles=n_tiles, clipped=not full, branch=branch)


def summary(p):
    return (p["block_n"], p["kbytes"], p["cluster"], p["b_resident"], p["epi"])


def check_plan(p, expect, sms):
    """the case's expected (block_n, kbytes, cluster, b_resident, epilogue); b_resident depends on the SM count and is
    only pinned for the 132-SM part."""
    got = summary(p)
    if sms != SMS:
        got, expect = got[:3] + got[4:], tuple(expect[:3]) + tuple(expect[4:])
    assert got == tuple(expect), "launch plan moved: %s, expected %s" % (got, expect)


# ---------------------------------------------------------------------------------------------------------------
# case tables (inference shapes: batch 8 at 416 px unless the name says otherwise)
# ---------------------------------------------------------------------------------------------------------------
# cin = real input channels, ck = channels of the K view; r = log2(out_scale / acc_scale); acc "np2": an acc_scale
# that is not a power of two; out "f32" = a head's fp32 rows in a 256-wide buffer, requant False = no fake-quant
Q = namedtuple("Q", "B H W cin ck cout k s layout act slope bias out requant r acc expect")
CASES = {
    # yolov3's layer 1 and layer 3, the two narrow layers layout.pair_form pairs
    "l1_c32-64_k3s2_416_s2pairs": Q(8, 416, 416, 32, 32, 64, 3, 2, "s2", "leaky", 0.1, True, "i8", True, 4, "pow2",
                                    (64, 64, 1, True, "i8-tma")),
    "l3_c32-64_k3_208_s1pairs": Q(8, 208, 208, 32, 32, 64, 3, 1, "s1", "leaky", 0.1, True, "i8", True, 5, "pow2",
                                  (128, 64, 1, True, "i8-tma")),
    # yolov3-tiny's 16-channel layer read through its zero-padded 32-channel K view
    "c16v32-32_k3_208": Q(8, 208, 208, 16, 32, 32, 3, 1, "dense", "leaky", 0.1, True, "i8", True, 3, "pow2",
                          (32, 32, 1, True, "i8-tma")),
    # 1x1 layers with more M tiles than SMs
    "c64-32_k1_208_nobias": Q(8, 208, 208, 64, 64, 32, 1, 1, "dense", "leaky", 0.125, False, "i8", True, 4, "pow2",
                              (32, 64, 1, True, "i8-tma")),
    "c128-64_k1_104": Q(8, 104, 104, 128, 128, 64, 1, 1, "dense", "leaky", 0.1, True, "i8", True, 6, "pow2",
                        (64, 128, 1, True, "i8-tma")),
    "c128-32_k3_26_nobias_linear": Q(8, 26, 26, 128, 128, 32, 3, 1, "dense", "linear", 0.1, False, "i8", True, 5,
                                     "pow2", (32, 128, 1, False, "i8-tma")),
    # 43 and 11 M tiles, odd, under the 2-CTA weight-multicast cluster; the 13-px layer with |acc| > 2^24
    "c256-512_k3s2_52": Q(8, 52, 52, 256, 256, 512, 3, 2, "dense", "leaky", 0.1, True, "i8", True, 6, "pow2",
                          (128, 128, 2, False, "i8-tma")),
    "c512-1024_k3_13_adversarial": Q(8, 13, 13, 512, 512, 1024, 3, 1, "dense", "leaky", 0.1, True, "i8", True, 6,
                                     "pow2", (128, 128, 2, False, "i8-tma")),
    # 32-byte k-steps; partial last N tiles into a channel slot: the general epilogue's int8 byte stores
    "c96-40_k3_52_slot": Q(8, 52, 52, 96, 96, 40, 3, 1, "dense", "leaky", 0.25, True, "i8", True, 4, "pow2",
                           (64, 32, 1, True, "general")),
    "c160-80_k1_26_slot": Q(8, 26, 26, 160, 160, 80, 1, 1, "dense", "leaky", 0.1, True, "i8", True, 3, "pow2",
                            (128, 32, 1, False, "general")),
    "c64-64_k1_104_hswish": Q(8, 104, 104, 64, 64, 64, 1, 1, "dense", "h_swish", 0.1, True, "i8", True, 3, "pow2",
                              (64, 64, 1, True, "general")),
    # acc * acc_scale rounds before the bias is added: the general path's two roundings
    "c128-128_k1_104_np2acc": Q(8, 104, 104, 128, 128, 128, 1, 1, "dense", "leaky", 0.1, True, "i8", True, 4, "np2",
                                (128, 128, 2, False, "general")),
    # fp32 heads in a 256-wide buffer: 255 columns end inside a 16-byte piece (general), 252 end on one (TMA clip)
    "head_c256-255_k1_52": Q(8, 52, 52, 256, 256, 255, 1, 1, "dense", "linear", 0.1, True, "f32", True, 4, "pow2",
                             (128, 128, 2, False, "general")),
    "head_c256-252_k1_52": Q(8, 52, 52, 256, 256, 252, 1, 1, "dense", "linear", 0.1, True, "f32", True, 4, "pow2",
                             (128, 128, 2, False, "f32-tma-fq")),
    "head_c256-252_k1_13_b2_raw": Q(2, 13, 13, 256, 256, 252, 1, 1, "dense", "linear", 0.1, True, "f32", False, 4,
                                    "pow2", (128, 128, 1, False, "f32-tma-linear")),
}
ADVERSARIAL = {"c512-1024_k3_13_adversarial"}

# the folded shortcut: conv shapes (out_scale 2^-4) x scale sets (a_in, scale_x, scale_a, scale_sum, clamp, branch)
SC_OUT_SCALE = 2.0 ** -4
SC_SHAPES = {
    "l3_c32-64_k3_208_s1pairs": CASES["l3_c32-64_k3_208_s1pairs"],
    "c64-128_k3_104": Q(8, 104, 104, 64, 64, 128, 3, 1, "dense", "leaky", 0.1, True, "i8", True, 4, "pow2",
                        (128, 64, 1, True, "i8-tma")),
    "c128-256_k3_52": Q(8, 52, 52, 128, 128, 256, 3, 1, "dense", "leaky", 0.1, True, "i8", True, 4, "pow2",
                        (128, 128, 2, False, "i8-tma")),
}
SC_BRANCHES = {
    # q / 2 + a: both roundings identities
    "simple": (2.0 ** -3, 2.0 ** -5, 2.0 ** -4, 2.0 ** -3, 0, "simple"),
    # rha(q / 2) + rha(a / 2) / 2: scale_x coarser than out_scale, scale_a coarser than a_in
    "rounded": (2.0 ** -5, 2.0 ** -3, 2.0 ** -4, 2.0 ** -3, 0, "rounded"),
    # google QuantizedShortcut_max: 2q and 2a clamped, then added and clamped
    "clamp": (2.0 ** -4, 2.0 ** -5, 2.0 ** -5, 2.0 ** -5, 1, "clamp"),
    # out_scale / scale_sum on both sides of the 4096 bound of the simple branch
    "cx4096": (2.0 ** -16, 2.0 ** -5, 2.0 ** -17, 2.0 ** -16, 0, "simple"),
    "cx8192": (2.0 ** -17, 2.0 ** -5, 2.0 ** -18, 2.0 ** -17, 0, "rounded"),
}


def _case_plan(c, sms, aligned=True, qres=None, dense_input=True):
    geo = int8_geometry(c.B, c.H, c.W, c.ck, c.cout, c.k, c.s, c.layout, dense_input)
    if geo is None:
        return None
    M, Cg, nout, ntaps = geo
    return int8_launch_plan(M, Cg, nout, ntaps, sms, out=c.out, act=c.act, slope=c.slope, acc_pow2=c.acc == "pow2",
                            requant=c.requant, aligned=aligned, qres=qres)


def _qres(a_in, sx, sa, ssum, clamp, out_scale=SC_OUT_SCALE, aligned=True):
    return dict(out_scale=out_scale, a_in=a_in, sx=sx, sa=sa, ssum=ssum, lo=-128, hi=127, clamp=clamp, aligned=aligned)


def test_int8_case_table_covers_every_launch_path():
    """Runs without a GPU: every case lands on the plan it names, and together they reach every launch variant."""
    plans = []
    for c in CASES.values():
        p = _case_plan(c, SMS)
        check_plan(p, c.expect, SMS)
        plans.append(p)
    branches = set()
    for c in SC_SHAPES.values():
        for (a_in, sx, sa, ssum, clamp, br) in SC_BRANCHES.values():
            p = _case_plan(c, SMS, qres=_qres(a_in, sx, sa, ssum, clamp))
            check_plan(p, c.expect, SMS)
            assert p["branch"] == br
            branches.add(br)
            plans.append(p)
    pairs = {(bn, kb) for bn in (32, 64, 128) for kb in (32, 64, 128)}
    assert {(p["block_n"], p["kbytes"]) for p in plans if p["cluster"] == 1} == pairs
    assert any(p["cluster"] == 2 and p["num_m_tiles"] % 2 == 1 for p in plans)
    assert {p["b_resident"] for p in plans} == {True, False}
    assert {p["epi"] for p in plans} == {"i8-tma", "f32-tma-fq", "f32-tma-linear", "general"}
    assert any(c.out == "i8" and p["clipped"] for c, p in zip(CASES.values(), plans))
    assert any(c.acc == "np2" for c in CASES.values())
    assert {c.act for c in CASES.values()} & {"relu6", "h_swish"}
    assert {c.bias for c in CASES.values()} == {True, False}
    assert branches == {"simple", "rounded", "clamp"}
    assert {c.layout for c in CASES.values()} == {"dense", "s1", "s2"}
    assert {c.layout for c in SC_SHAPES.values()} >= {"s1"}
    assert any(p["cluster"] == 2 for c in SC_SHAPES.values() for p in [_case_plan(c, SMS)])
    # the simple branch's bounds, on both sides of each

    def q(cx, ca):
        ssum = SC_OUT_SCALE / cx
        return _case_plan(SC_SHAPES["c64-128_k3_104"], SMS,
                          qres=_qres(ca * ssum, SC_OUT_SCALE, ca * ssum, ssum, 0))["branch"]

    assert [q(4096, 1), q(8192, 1), q(1, 4096), q(1, 8192)] == ["simple", "rounded", "simple", "rounded"]
    assert [q(2.0 ** -12, 1), q(2.0 ** -13, 1), q(1, 2.0 ** -12), q(1, 2.0 ** -13)] == \
        ["simple", "rounded", "simple", "rounded"]
    # the refusals exercised by test_int8_refusals_are_errors and test_qconv_shortcut_refusals_leave_output
    tiny = CASES["c16v32-32_k3_208"]
    assert _case_plan(tiny._replace(ck=16), SMS) is None                                 # 16-byte K
    assert _case_plan(CASES["l1_c32-64_k3s2_416_s2pairs"], SMS, dense_input=False) is None   # pair view of a slice
    sc = SC_SHAPES["c64-128_k3_104"]
    good = SC_BRANCHES["simple"][:5]
    assert _case_plan(sc, SMS, qres=_qres(*good)) is not None
    assert _case_plan(sc, SMS, qres=_qres(*good[:1], 3 * 2.0 ** -7, *good[2:])) is None       # scale_x not 2^n
    assert _case_plan(sc, SMS, qres=_qres(*good, aligned=False)) is None                     # addend alignment
    assert _case_plan(sc._replace(acc="np2"), SMS, qres=_qres(*good)) is None                # general epilogue
    assert _case_plan(CASES["c160-80_k1_26_slot"], SMS, qres=_qres(*good)) is None           # partial N tile


# ---------------------------------------------------------------------------------------------------------------
# the oracle (plain fp32 torch ops, one per rounding; scalars as fp32 tensors so no op turns a division into a
# multiplication by a reciprocal)
# ---------------------------------------------------------------------------------------------------------------
def _f32(v, dev):
    return torch.tensor(v, dtype=torch.float32, device=dev)


def _act32(v, act, slope):
    if act == "leaky":
        return torch.where(v > 0, v, v * _f32(slope, v.device))
    if act == "relu6":
        return v.clamp(0.0, 6.0)
    if act == "h_swish":
        return v * ((v + 3.0).clamp(0.0, 6.0) / _f32(6.0, v.device))
    assert act == "linear"
    return v


def requant_oracle(acc64, acc_scale, bias, act, slope, out_scale, lo=-128, hi=127):
    """(v, codes, counts) of act(acc * acc_scale + bias) requantised onto out_scale; acc64 NCHW fp64"""
    dev = acc64.device
    v = acc64.float() * _f32(acc_scale, dev)
    if bias is not None:
        v = v + bias.view(1, -1, 1, 1)
    v = _act32(v, act, slope)
    t = v * _f32(1.0 / out_scale, dev)
    r = orc.round_half_away(t)
    tie = ((t.abs() - t.abs().floor()) == 0.5) & (r >= lo) & (r <= hi)
    counts = dict(tie_pos=int((tie & (t > 0)).sum()), tie_neg=int((tie & (t < 0)).sum()),
                  sat_lo=int((r < lo).sum()), sat_hi=int((r > hi).sum()))
    return v, r.clamp(lo, hi), counts


def shortcut_oracle(x, sx_in, a, sa_in, sx, sa, ssum, lo=-128, hi=127, clamp=False):
    """clamp(rha((rha(x*sx_in/sx)*sx + rha(a*sa_in/sa)*sa) / ssum)), the addends clamped too in clamp mode"""
    dev = x.device
    f = lambda v: _f32(v, dev)
    xr = orc.round_half_away(x.float() * f(sx_in) / f(sx))
    ar = orc.round_half_away(a.float() * f(sa_in) / f(sa))
    if clamp:
        xr, ar = xr.clamp(lo, hi), ar.clamp(lo, hi)
    return orc.round_half_away((xr * f(sx) + ar * f(sa)) / f(ssum)).clamp(lo, hi)


def _nhwc8(t):
    return t.permute(0, 2, 3, 1).to(torch.int8)


# ---------------------------------------------------------------------------------------------------------------
# case data (device-agnostic)
# ---------------------------------------------------------------------------------------------------------------
def _seed(name):
    return zlib.crc32(name.encode()) % 10007


def _codes(g, shape, dev):
    return torch.randint(-128, 128, shape, generator=g, device=dev, dtype=torch.int8)


def _extreme_codes(g, shape, dev):
    """+127 / -128 at random: the codes a launch must never read (or must read through zero weights)"""
    return torch.where(torch.rand(shape, generator=g, device=dev) < 0.5, 127, -128).to(torch.int8)


def _out_scale(c):
    return OUT_SCALE_HSWISH if c.act == "h_swish" else OUT_SCALE


def _spread(c):
    """standard deviation of (acc + bias) / 2^r that puts both ends of [-128, 127] in reach after the activation"""
    if c.act == "leaky":
        return 100.0 / c.slope
    if c.act == "h_swish":
        return 1.5 / OUT_SCALE_HSWISH   # v ~ +-1.5: the curved part, saturating above v ~ 0.45
    return 100.0


def _acc_scale(c, out_scale):
    s = out_scale / 2.0 ** c.r
    return float(torch.tensor(s * 1.1, dtype=torch.float32)) if c.acc == "np2" else s


def make_case(c, name, dev, out_scale=None):
    """x (the real channels, NHWC int8), xv (the view the launch reads), OIHW weight codes (float), fp32 bias"""
    g = torch.Generator(device=dev).manual_seed(_seed(name))
    if c.layout == "dense":
        xbuf = _extreme_codes(g, (c.B, c.H, c.W, LEAD + c.ck + TRAIL), dev)
        xbuf[..., LEAD:LEAD + c.cin] = _codes(g, (c.B, c.H, c.W, c.cin), dev)
        xv = xbuf[..., LEAD:LEAD + c.ck]
    else:
        xv = _codes(g, (c.B, c.H, c.W, c.cin), dev)
    x = xv[..., :c.cin]
    out_scale = out_scale or _out_scale(c)
    sigma = _spread(c) * 2.0 ** c.r / ((c.cin * c.k * c.k) ** 0.5 * 73.9)
    w = (torch.randn(c.cout, c.cin, c.k, c.k, generator=g, device=dev) * sigma).round().clamp(-128, 127)
    if name in ADVERSARIAL:
        # one +-127 / -128 code per input channel, flipped at 10 % of the pixels; output channel 0 has the same signs as
        # weights, channel 1 the opposite: |acc| ~ 0.8 * 4608 * 127 * 128 > 2^24 inside the border
        pat = _extreme_codes(g, (c.cin,), dev)
        flip = torch.rand((c.B, c.H, c.W, c.cin), generator=g, device=dev) < 0.1
        x.copy_(torch.where(flip, _extreme_codes(g, (c.B, c.H, c.W, c.cin), dev), pat.view(1, 1, 1, -1)))
        w[0] = pat.float().view(-1, 1, 1)
        w[1] = torch.where(pat < 0, 127.0, -128.0).view(-1, 1, 1)
    acc_scale = _acc_scale(c, out_scale)
    bias = None
    if c.bias:
        span = 64 * 2 ** c.r
        bias = (torch.randint(-span, span, (c.cout,), generator=g, device=dev).float() * (out_scale / 2.0 ** c.r))
    return x, xv, w, bias, acc_scale


def case_oracle(c, x, w, bias, acc_scale, out_scale=None):
    out_scale = out_scale or _out_scale(c)
    pad = (c.k - 1) // 2
    acc = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=c.s, padding=pad)
    v, q, counts = requant_oracle(acc, acc_scale, bias, c.act, c.slope, out_scale)
    counts["max_acc"] = float(acc.abs().max())
    return v, q, counts


# ---------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------
def _ops():
    from b200yolo import ops
    return ops


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pack_dense(w, ck):
    """[O][k][k][ck] int8 with zero columns at the view's pad channels"""
    O, I, k, _ = w.shape
    wp = torch.zeros((O, k, k, ck), dtype=torch.int8, device=w.device)
    wp[..., :I] = w.permute(0, 2, 3, 1).to(torch.int8)
    return wp


def _pairs(t):
    B, H, W, Cc = t.shape
    return t.view(B, H, W // 2, 2 * Cc)


class _Margins:
    """a dense NHWC tensor between two sentinel margins of a flat buffer (the pair views need dense tensors)"""
    PAD = 4096

    def __init__(self, shape, dtype, sentinel, dev):
        n = 1
        for d in shape:
            n *= d
        self.n, self.sentinel = n, sentinel
        self.flat = torch.full((n + 2 * self.PAD,), sentinel, dtype=dtype, device=dev)
        self.t = self.flat[self.PAD:self.PAD + n].view(shape)

    def untouched(self):
        return bool((self.flat[:self.PAD] == self.sentinel).all()) and bool((self.flat[self.PAD + self.n:] ==
                                                                              self.sentinel).all())


def _slot(shape_bhw, cout, dtype, sentinel, lead, trail, dev):
    buf = torch.full(tuple(shape_bhw) + (lead + cout + trail,), sentinel, dtype=dtype, device=dev)
    return buf, buf[..., lead:lead + cout]


def _slot_untouched(buf, lead, n, sentinel):
    return bool((buf[..., :lead] == sentinel).all()) and bool((buf[..., lead + n:] == sentinel).all())


def _weights_for(c, w, bias, ops):
    """(QConvPack.w8, QConvPack.bias, w_layout) as qengine.QPlan._pack_qconv lays them out for the case's form"""
    from b200yolo.lib import WLAYOUT_S2_PAIRS
    if c.layout == "s2":
        return ops.s2_pair_weights(w).to(torch.int8).contiguous(), bias, WLAYOUT_S2_PAIRS
    if c.layout == "s1":
        w2 = ops.s1_pair_weights(w)
        return w2.permute(0, 2, 3, 1).to(torch.int8).contiguous(), torch.cat([bias, bias]).contiguous(), 0
    return _pack_dense(w, c.ck), bias, 0


def _print_case(tag, p, **numbers):
    keys = ("block_n", "kbytes", "cluster", "b_resident", "epi", "num_m_tiles", "num_n_tiles", "branch")
    print("\n%s: %s %s" % (tag, " ".join("%s=%s" % (k, p[k]) for k in keys),
                           " ".join("%s=%s" % kv for kv in numbers.items())))


# ---------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_int8_conv_forward_against_integer_oracle(name):
    from b200yolo.lib import OUT_F32, OUT_I8
    c = CASES[name]
    ops = _ops()
    dev = "cuda"
    x, xv, w, bias, acc_scale = make_case(c, name, dev)
    pad = (c.k - 1) // 2
    Ho, Wo = (c.H + 2 * pad - c.k) // c.s + 1, (c.W + 2 * pad - c.k) // c.s + 1
    w8, b8, layout = _weights_for(c, w, bias, ops)
    out_scale = _out_scale(c)
    p = _case_plan(c, _sms())
    check_plan(p, c.expect, _sms())

    if c.layout == "s1":
        m = _Margins((c.B, Ho, Wo, c.cout), torch.int8, SENT8, dev)
        ops.qconv2d(_pairs(xv), w8, b8, 3, 1, 1, acc_scale, out_scale, act=c.act, slope=c.slope, out=_pairs(m.t),
                    out_kind=OUT_I8)
        got, untouched = m.t, m.untouched
    elif c.out == "i8":
        buf, ov = _slot((c.B, Ho, Wo), c.cout, torch.int8, SENT8, LEAD, TRAIL, dev)
        ops.qconv2d(xv, w8, b8, c.k, c.s, pad, acc_scale, out_scale, act=c.act, slope=c.slope, out=ov,
                    out_kind=OUT_I8, w_layout=layout)
        got, untouched = ov, lambda: _slot_untouched(buf, LEAD, c.cout, SENT8)
    else:
        buf, ov = _slot((c.B, Ho, Wo), c.cout, torch.float32, SENT32, 0, 256 - c.cout, dev)
        ops.qconv2d(xv, w8, b8, c.k, c.s, pad, acc_scale, out_scale, act=c.act, slope=c.slope, out=ov,
                    out_kind=OUT_F32, requant=c.requant)
        got, untouched = ov, lambda: _slot_untouched(buf, 0, c.cout, SENT32)
    v, q, counts = case_oracle(c, x, w, bias, acc_scale)
    if c.out == "i8":
        want = _nhwc8(q)
    else:
        want = (q * _f32(out_scale, dev) if c.requant else v).permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    diff = int((got != want).sum())
    _print_case(name, p, **counts, mismatches=diff)
    assert untouched(), "wrote outside the output slot"
    assert diff == 0, "%d of %d outputs differ from the integer oracle" % (diff, want.numel())
    if c.requant:
        # the rounding rule and the clamp were exercised, on both sides (h_swish never reaches the lowest code at a
        # scale where it has ties, OUT_SCALE_HSWISH)
        need = ("tie_pos", "tie_neg", "sat_hi") + (() if c.act == "h_swish" else ("sat_lo",))
        assert min(counts[k] for k in need) > 0, counts
    if name in ADVERSARIAL:
        assert counts["max_acc"] > 2 ** 24


@pytest.mark.gpu
def test_int8_refusals_are_errors():
    """int8 launches the kernel cannot run are B2YError and write nothing"""
    from b200yolo.lib import B2YError, OUT_I8, WLAYOUT_S2_PAIRS
    ops = _ops()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(3)
    # 16 channels: 16-byte k-steps
    x16 = _codes(g, (2, 20, 20, 16), dev)
    out = torch.full((2, 20, 20, 32), SENT8, dtype=torch.int8, device=dev)
    with pytest.raises(B2YError):
        ops.qconv2d(x16, torch.zeros((32, 3, 3, 16), dtype=torch.int8, device=dev), None, 3, 1, 1, 2.0 ** -12,
                    OUT_SCALE, out=out, out_kind=OUT_I8)
    # the stride-2 pixel-pair view of a channel slice (in_pitch != in_c)
    xb = _codes(g, (2, 20, 20, 64), dev)
    out2 = torch.full((2, 10, 10, 64), SENT8, dtype=torch.int8, device=dev)
    with pytest.raises(B2YError):
        ops.qconv2d(xb[..., :32], torch.zeros((64, 3, 2, 64), dtype=torch.int8, device=dev), None, 3, 2, 1,
                    2.0 ** -12, OUT_SCALE, out=out2, out_kind=OUT_I8, w_layout=WLAYOUT_S2_PAIRS)
    torch.cuda.synchronize()
    assert bool((out == SENT8).all()) and bool((out2 == SENT8).all())


# ---------------------------------------------------------------------------------------------------------------
# the shortcut folded into the conv epilogue
# ---------------------------------------------------------------------------------------------------------------
def _call(name, *args):
    from b200yolo.lib import call
    call(name, *args)


def _qshortcut(x, sx_in, a, sa_in, out, c, sx, sa, ssum, lo=-128.0, hi=127.0):
    from b200yolo.lib import ptr, stream_ptr
    ops = _ops()
    pixels = x.shape[0] * x.shape[1] * x.shape[2]
    _call("b2y_qshortcut_i8", ptr(x), ops._pitch(x), ptr(a), ops._pitch(a), ptr(out), ops._pitch(out), pixels, c,
          sx_in, sx, sa_in, sa, ssum, lo, hi, stream_ptr())


def _requant(x, out, c, s_in, s_out, lo=-128.0, hi=127.0):
    from b200yolo.lib import ptr, stream_ptr
    ops = _ops()
    pixels = x.shape[0] * x.shape[1] * x.shape[2]
    _call("b2y_requant_i8", ptr(x), ops._pitch(x), ptr(out), ops._pitch(out), pixels, c, s_in, s_out, lo, hi,
          stream_ptr())


def _qconv_shortcut(xv, w8, bias, k, s, pad, act, slope, acc_scale, out_scale, av, a_pitch, a_in, sx, sa, ssum,
                    clamp, ov, layout=0):
    from b200yolo.lib import OUT_I8, QConvDesc, ptr, stream_ptr
    ops = _ops()
    cd = ops.make_conv_desc(xv.shape, ops._pitch(xv), w8.shape[0], k, s, pad, ops._pitch(ov), act, slope, OUT_I8, 0,
                            layout)
    qd = QConvDesc(cd, float(acc_scale), float(out_scale), -128.0, 127.0, OUT_I8, 1, clamp)
    _call("b2y_qconv2d_shortcut_fwd", C.byref(qd), ptr(xv), ptr(w8), ptr(bias), ptr(av), a_pitch, a_in, sx, sa, ssum,
          -128.0, 127.0, ptr(ov), stream_ptr())


def _shortcut_setup(name, dev):
    """the conv of SC_SHAPES[name], its oracle codes (NHWC) and the addend (NHWC codes + the view the launch reads,
    a slice of a wider buffer: qres_pitch != C)"""
    c = SC_SHAPES[name]
    ops = _ops()
    x, xv, w, bias, acc_scale = make_case(c, name, dev, SC_OUT_SCALE)
    pad = (c.k - 1) // 2
    Ho, Wo = (c.H + 2 * pad - c.k) // c.s + 1, (c.W + 2 * pad - c.k) // c.s + 1
    w8, b8, layout = _weights_for(c, w, bias, ops)
    _, q, _ = case_oracle(c, x, w, bias, acc_scale, SC_OUT_SCALE)
    g = torch.Generator(device=dev).manual_seed(_seed(name) + 1)
    if c.layout == "s1":
        abuf = _extreme_codes(g, (c.B, Ho, Wo // 2, 2 * c.cout + 32), dev)
        av = abuf[..., :2 * c.cout]
        av.copy_(_codes(g, av.shape, dev))
        a = av.reshape(c.B, Ho, Wo, c.cout)
    else:
        abuf = _extreme_codes(g, (c.B, Ho, Wo, c.cout + 32), dev)
        av = abuf[..., 16:16 + c.cout]
        av.copy_(_codes(g, av.shape, dev))
        a = av
    return c, xv, w8, b8, layout, acc_scale, _nhwc8(q), a, av, abuf.shape[-1], (Ho, Wo)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SC_SHAPES))
def test_qconv_shortcut_every_branch_against_oracle(name):
    """b2y_qconv2d_shortcut_fwd in each branch == the oracle == qconv2d + b2y_qshortcut_i8 (+ b2y_requant_i8 of both
    addends in clamp mode, as qengine runs it unfused)"""
    from b200yolo.lib import OUT_I8
    ops = _ops()
    dev = "cuda"
    c, xv, w8, b8, layout, acc_scale, q, a, av, a_pitch, (Ho, Wo) = _shortcut_setup(name, dev)
    pad = (c.k - 1) // 2
    pairs = c.layout == "s1"
    for br, (a_in, sx, sa, ssum, clamp, branch) in SC_BRANCHES.items():
        p = _case_plan(c, _sms(), qres=_qres(a_in, sx, sa, ssum, clamp))
        check_plan(p, c.expect, _sms())
        assert p["branch"] == branch
        want = shortcut_oracle(q, SC_OUT_SCALE, a, a_in, sx, sa, ssum, clamp=bool(clamp))
        # fused
        if pairs:
            m = _Margins((c.B, Ho, Wo, c.cout), torch.int8, SENT8, dev)
            _qconv_shortcut(_pairs(xv), w8, b8, 3, 1, 1, c.act, c.slope, acc_scale, SC_OUT_SCALE, av, a_pitch, a_in,
                            sx, sa, ssum, clamp, _pairs(m.t))
            fused, untouched = m.t, m.untouched
        else:
            buf, ov = _slot((c.B, Ho, Wo), c.cout, torch.int8, SENT8, LEAD, TRAIL, dev)
            _qconv_shortcut(xv, w8, b8, c.k, c.s, pad, c.act, c.slope, acc_scale, SC_OUT_SCALE, av, a_pitch, a_in, sx,
                            sa, ssum, clamp, ov, layout)
            fused, untouched = ov, (lambda buf=buf: _slot_untouched(buf, LEAD, c.cout, SENT8))
        # unfused: the conv's own codes, then the stand-alone shortcut
        own = torch.empty((c.B, Ho, Wo, c.cout), dtype=torch.int8, device=dev)
        xs = _pairs(xv) if pairs else xv
        ops.qconv2d(xs, w8, b8, c.k, c.s, pad, acc_scale, SC_OUT_SCALE, act=c.act, slope=c.slope,
                    out=_pairs(own) if pairs else own, out_kind=OUT_I8, w_layout=layout)
        sep = torch.empty_like(own)
        ow, sepv = (_pairs(own), _pairs(sep)) if pairs else (own, sep)
        cc = ow.shape[3]
        x_in, sx_in, a_src, sa_src = ow, SC_OUT_SCALE, av, a_in
        if clamp:
            tmp = torch.empty((2,) + tuple(ow.shape), dtype=torch.int8, device=dev)
            _requant(ow, tmp[0], cc, SC_OUT_SCALE, sx)
            _requant(av, tmp[1], cc, a_in, sa)
            x_in, sx_in, a_src, sa_src = tmp[0], sx, tmp[1], sa
        _qshortcut(x_in, sx_in, a_src, sa_src, sepv, cc, sx, sa, ssum)
        torch.cuda.synchronize()
        assert torch.equal(own, q), "%s: the conv codes differ from the oracle" % br
        d_f, d_s = int((fused != want).sum()), int((sep != want).sum())
        w32 = want.float()
        _print_case("%s %s" % (name, br), p, fused_mismatch=d_f, unfused_mismatch=d_s,
                    sat_lo=int((w32 == -128).sum()), sat_hi=int((w32 == 127).sum()))
        assert untouched(), "%s: wrote outside the output" % br
        assert d_f == 0, "%s: fused shortcut differs from the oracle in %d of %d codes" % (br, d_f, want.numel())
        assert d_s == 0, "%s: qconv2d + b2y_qshortcut_i8 differ from the oracle in %d codes" % (br, d_s)


@pytest.mark.gpu
def test_qconv_shortcut_refusals_leave_output():
    """a scale that is not a power of two, an accumulator scale that is not one either, a misaligned addend or one
    whose pitch is not a multiple of 16: B2YError 'unsupported', nothing launched, the output keeps its bytes"""
    from b200yolo.lib import B2YError
    dev = "cuda"
    name = "c64-128_k3_104"
    c, xv, w8, b8, layout, acc_scale, q, a, av, a_pitch, (Ho, Wo) = _shortcut_setup(name, dev)
    a_in, sx, sa, ssum, clamp, _ = SC_BRANCHES["simple"]
    g = torch.Generator(device=dev).manual_seed(4)
    flat = _codes(g, (c.B * Ho * Wo * a_pitch + 64,), dev)
    misaligned = flat[1:1 + c.B * Ho * Wo * a_pitch].view(c.B, Ho, Wo, a_pitch)[..., :c.cout]
    narrow = _codes(g, (c.B, Ho, Wo, c.cout + 8), dev)[..., :c.cout]
    bad = {
        "scale_x 3 * 2^-7": dict(sx=3 * 2.0 ** -7),
        "acc_scale not 2^n": dict(acc=acc_scale * 1.5),
        "addend misaligned": dict(av=misaligned, a_pitch=a_pitch),
        "addend pitch 136": dict(av=narrow, a_pitch=c.cout + 8),
    }
    buf, ov = _slot((c.B, Ho, Wo), c.cout, torch.int8, SENT8, LEAD, TRAIL, dev)
    for why, b in bad.items():
        with pytest.raises(B2YError, match="(?i)unsupported"):
            _qconv_shortcut(xv, w8, b8, c.k, c.s, 1, c.act, c.slope, b.get("acc", acc_scale), SC_OUT_SCALE,
                            b.get("av", av), b.get("a_pitch", a_pitch), a_in, b.get("sx", sx), sa, ssum, clamp, ov)
    torch.cuda.synchronize()
    assert bool((buf == SENT8).all()), "a refused launch wrote"


# ---------------------------------------------------------------------------------------------------------------
# the other int8 kernels
# ---------------------------------------------------------------------------------------------------------------
# C = 48 / 80 / 96: 256 % (C / 16) != 0 takes the v1 kernel; a scale that is not 2^n takes v2's divisions
QSC_CASES = {
    "v2_exact_c64": (64, (2.0 ** -4, 2.0 ** -3, 2.0 ** -5, 2.0 ** -4, 2.0 ** -3)),
    "v2_div_c64": (64, (2.0 ** -4, 3 * 2.0 ** -6, 2.0 ** -5, 5 * 2.0 ** -8, 3 * 2.0 ** -5)),
    "v1_c48": (48, (2.0 ** -4, 2.0 ** -3, 2.0 ** -5, 2.0 ** -4, 2.0 ** -3)),
    "v1_c80": (80, (2.0 ** -3, 2.0 ** -5, 2.0 ** -4, 2.0 ** -6, 2.0 ** -4)),
    "v1_c96_div": (96, (2.0 ** -4, 3 * 2.0 ** -6, 2.0 ** -5, 5 * 2.0 ** -8, 3 * 2.0 ** -5)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(QSC_CASES))
def test_qshortcut_i8_against_oracle(name):
    """b2y_qshortcut_i8 (v2<exact>, v2<div>, v1) from addends in wider buffers into a channel slot"""
    dev = "cuda"
    cc, (sx_in, sx, sa_in, sa, ssum) = QSC_CASES[name]
    g = torch.Generator(device=dev).manual_seed(_seed(name))
    B, H, W = 4, 52, 52
    xb = _extreme_codes(g, (B, H, W, cc + 32), dev)
    ab = _extreme_codes(g, (B, H, W, cc + 48), dev)
    x, a = xb[..., 16:16 + cc], ab[..., 32:32 + cc]
    x.copy_(_codes(g, x.shape, dev))
    a.copy_(_codes(g, a.shape, dev))
    buf, ov = _slot((B, H, W), cc, torch.int8, SENT8, LEAD, TRAIL, dev)
    _qshortcut(x, sx_in, a, sa_in, ov, cc, sx, sa, ssum)
    want = shortcut_oracle(x, sx_in, a, sa_in, sx, sa, ssum)
    torch.cuda.synchronize()
    d = int((ov != want).sum())
    print("\n%s: mismatches %d, saturated %d / %d" % (name, d, int((want == -128).sum()), int((want == 127).sum())))
    assert _slot_untouched(buf, LEAD, cc, SENT8)
    assert d == 0, "%d of %d codes differ" % (d, want.numel())


REQUANT_CASES = {
    "identity": (2.0 ** -5, 2.0 ** -5, -128, 127),
    "up_saturating": (2.0 ** -5, 2.0 ** -7, -128, 127),
    "down_ties": (2.0 ** -5, 2.0 ** -3, -128, 127),
    "not_pow2": (2.0 ** -5, 3 * 2.0 ** -7, -128, 127),
    "bits4": (2.0 ** -5, 2.0 ** -4, -8, 7),
}


@pytest.mark.gpu
def test_requant_i8_against_oracle():
    """b2y_requant_i8 into a concat slot: a copy, codes scaled up (saturating), down (ties), by a scale that is not a
    power of two, and onto 4-bit bounds"""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(31)
    B, H, W, cc = 4, 26, 26, 96
    xb = _extreme_codes(g, (B, H, W, cc + 32), dev)
    x = xb[..., 16:16 + cc]
    x.copy_(_codes(g, x.shape, dev))
    for name, (s_in, s_out, lo, hi) in REQUANT_CASES.items():
        buf, ov = _slot((B, H, W), cc, torch.int8, SENT8, 128, 64, dev)
        _requant(x, ov, cc, s_in, s_out, float(lo), float(hi))
        want = orc.round_half_away(x.float() * _f32(s_in, dev) / _f32(s_out, dev)).clamp(lo, hi)
        torch.cuda.synchronize()
        assert _slot_untouched(buf, 128, cc, SENT8), name
        assert torch.equal(ov, want.to(torch.int8)), "%s: %d codes differ" % (name, int((ov != want).sum()))
    assert torch.equal(ov.float().unique().sort().values, torch.arange(-8.0, 8.0, device=dev))


@pytest.mark.gpu
def test_upsample_nearest_i8_into_concat_slot():
    """yolov3's upsample: 13 x 13 x 256 codes to 26 x 26, into channels [0, 256) of the 768-wide route buffer whose
    other channels keep their bytes"""
    from b200yolo.lib import ptr, stream_ptr
    ops = _ops()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(41)
    B, H, W, cc = 8, 13, 13, 256
    xb = _extreme_codes(g, (B, H, W, cc + 32), dev)
    x = xb[..., :cc]
    x.copy_(_codes(g, x.shape, dev))
    for scale, lead in ((2, 0), (3, 512)):
        buf, ov = _slot((B, H * scale, W * scale), cc, torch.int8, SENT8, lead, 768 - cc - lead, dev)
        _call("b2y_upsample_nearest_i8", ptr(x), ops._pitch(x), ptr(ov), ops._pitch(ov), B, H, W, cc, scale,
              stream_ptr())
        want = x.repeat_interleave(scale, dim=1).repeat_interleave(scale, dim=2)
        torch.cuda.synchronize()
        assert _slot_untouched(buf, lead, cc, SENT8)
        assert torch.equal(ov, want)


@pytest.mark.gpu
def test_pack_qconv_weights_ties_and_range():
    """b2y_pack_qconv_weights: exact .5 ties of both signs, values just below them, codes beyond the range (8 and
    4 bits), a scale that is not a power of two; [O][I][kh][kw] -> [O][kh][kw][I]"""
    ops = _ops()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(51)
    O, I, k = 64, 96, 3
    base = torch.randint(-150, 150, (O, I, k, k), generator=g, device=dev).float()
    frac = torch.tensor([0.0, 0.5, -0.5, 0.25, 0.49999997, -0.49999997, 0.75], device=dev)
    sel = torch.randint(0, len(frac), (O, I, k, k), generator=g, device=dev)
    codes = base + frac[sel]
    for bits, s_w in ((8, 2.0 ** -9), (4, 2.0 ** -6), (8, 3 * 2.0 ** -10)):
        w = codes * _f32(s_w, dev)
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        got = ops.pack_qconv_weights(w, s_w, bits)
        want = orc.round_half_away(w / _f32(s_w, dev)).clamp(lo, hi).permute(0, 2, 3, 1).to(torch.int8)
        torch.cuda.synchronize()
        assert torch.equal(got, want), "bits %d scale %g: %d codes differ" % (bits, s_w, int((got != want).sum()))
        if s_w == 2.0 ** -9:
            t = w / _f32(s_w, dev)
            assert bool((t.abs().frac() == 0.5).any() & (t > hi).any() & (t < lo).any())


STEM_CASES = {"s1_c3-32_416": (1, 32, 0.1), "s2_c3-64_416": (2, 64, 0.25)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STEM_CASES))
def test_int8_stems_against_oracle(name):
    """b2y_stem_conv_fwd_q (fp32 CUDA cores) and b2y_stem_conv_fwd_fused_q (fp16 tensor cores) on k / 256 images with
    fake-quantised weights (code x 2^-8) and a bias on the s_w grid: every product is a whole number of s_w / 256 in
    fp16 and fp32 and the 27-term sums stay below 2^20 of them, so both are exact in any order and equal the oracle"""
    from b200yolo.lib import OUT_I8, ptr, stream_ptr
    ops = _ops()
    dev = "cuda"
    s, cout, slope = STEM_CASES[name]
    g = torch.Generator(device=dev).manual_seed(_seed(name))
    B, H, W, s_w = 2, 416, 416, 2.0 ** -8
    x = torch.randint(0, 256, (B, 3, H, W), generator=g, device=dev).float() / 256.0
    wq = torch.randint(-128, 128, (cout, 3, 3, 3), generator=g, device=dev).float() * s_w
    bq = torch.randint(-128, 128, (cout,), generator=g, device=dev).float() * s_w
    unit = s_w / 256
    acc = F.conv2d(x.double(), wq.double(), bq.double(), stride=s, padding=1)
    assert float(acc.abs().max()) / unit < 2 ** 20
    out_scale = 64 * unit
    v = _act32(acc.float(), "leaky", slope)
    t = v * _f32(1.0 / out_scale, dev)
    r = orc.round_half_away(t)
    want = _nhwc8(r.clamp(-128, 127))
    tie = (t.abs().frac() == 0.5) & (r.abs() <= 127)
    counts = dict(tie_pos=int((tie & (t > 0)).sum()), tie_neg=int((tie & (t < 0)).sum()), sat_lo=int((r < -128).sum()),
                  sat_hi=int((r > 127).sum()))
    Ho, Wo = want.shape[1], want.shape[2]
    ws = ops.pack_stem_weights(wq)
    for kern in ("b2y_stem_conv_fwd_q", "b2y_stem_conv_fwd_fused_q"):
        buf, ov = _slot((B, Ho, Wo), cout, torch.int8, SENT8, 16, 16, dev)
        d = ops.make_conv_desc((B, H, W, 3), 3, cout, 3, s, 1, ops._pitch(ov), "leaky", slope, OUT_I8)
        if kern == "b2y_stem_conv_fwd_q":
            _call(kern, C.byref(d), ptr(x), ptr(wq), ptr(bq), ptr(ov), out_scale, -128.0, 127.0, stream_ptr())
        else:
            _call(kern, C.byref(d), ptr(x), 0, 1.0, ptr(ws), ptr(bq), ptr(ov), out_scale, -128.0, 127.0, stream_ptr())
        torch.cuda.synchronize()
        diff = int((ov != want).sum())
        print("\n%s %s: %s mismatches %d" % (name, kern, counts, diff))
        assert _slot_untouched(buf, 16, cout, SENT8)
        assert diff == 0, "%s: %d of %d codes differ" % (kern, diff, want.numel())
    assert min(counts.values()) > 0, counts


@pytest.mark.gpu
def test_qat_stem_with_tiny_weight_scale_is_exact():
    """A trained google-QAT model whose layer 0 is then scaled by 2^-22 (BatchNorm gamma and beta, and with them the
    weight, bias and activation scales, so its codes stay what they were): its fake-quantised weights lie below fp16's
    subnormal grid, which the fused fp16 stem cannot hold.  The INT8 graph's layer-0 codes must still be the exact ones:
    the oracle's on the fp64 conv, and b2y_stem_conv_fwd_q's on the same weights."""
    import test_gpu_qat_int8 as qi
    from b200yolo.lib import OUT_I8, ptr, stream_ptr
    ops = _ops()
    qm = qi._qat_model("yolov3", 1)
    qi._train(qm, 2)
    conv0 = qm.module_list[0][0]
    with torch.no_grad():
        conv0.gamma.mul_(2.0 ** -22)
        conv0.beta.mul_(2.0 ** -22)
        for qz in (conv0.weight_quantizer, conv0.bias_quantizer, conv0.activation_quantizer):
            qz.scale = qz.scale * 2.0 ** -22
    x = orc.synth_images(2, 64, 64, seed=5).cuda()
    qm.use_cuda_graph = False
    with torch.no_grad():
        qm(x)
    plan = qm.engine().plans[qi._q1_plans(qm)[0]]
    stem = plan.packed[0]
    wq, bq, s_a, act, slope = stem.w, stem.bias, stem.s_a, stem.act, stem.slope
    assert float(wq[wq != 0].abs().min()) < 2.0 ** -24, "the weights are not below fp16's subnormal grid"
    got = plan.steps[0].out.view()
    # k / 256 times code x 2^-n: every product and sum exact in fp64, and in fp32 (< 2^24 units of s_w / 256)
    acc = F.conv2d(x.double(), wq.double(), bq.double(), stride=1, padding=1)
    _, q, _ = requant_oracle(acc, 1.0, None, act, slope, s_a)
    direct = torch.full_like(got, SENT8)
    d = ops.make_conv_desc((2, 64, 64, 3), 3, conv0.out_channels, 3, 1, 1, ops._pitch(direct), act, slope, OUT_I8)
    _call("b2y_stem_conv_fwd_q", C.byref(d), ptr(x), ptr(wq), ptr(bq), ptr(direct), s_a, -128.0, 127.0, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(direct, _nhwc8(q)), "b2y_stem_conv_fwd_q differs from the oracle"
    assert torch.equal(got, _nhwc8(q)), "layer 0: %d of %d codes differ" % (int((got != _nhwc8(q)).sum()), got.numel())
