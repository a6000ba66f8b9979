"""Weight gradient (csrc/wgrad_tc.cu) accumulating into a pre-filled dW: one split-K slice (the kernel adds into dW) and
several (partial tiles reduced in a fixed order), for the general kernel at every N tile width and the tap-transposed
kernel at Cin 32 / 64.  Each case is checked against an fp64 reference, and repeated or concurrent runs must agree bit
for bit."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from b200yolo import ops
    return ops


def plan(B, H, W, Cin, Cout, k, stride, sms):
    """(kernel, N tile width, split-K slices, last slice shorter) as b2y_conv2d_bwd_weight chooses them."""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    ksteps = -(-B * Ho * Wo // 64)
    if k == 3 and Cin in (32, 64):
        kern, bn = "taps", 64 if Cin == 32 else 32
        sp = min(max(1, sms // -(-Cout // bn)), ksteps)
    else:
        kern = "general"
        bn = (128 if Cin >= 128 else 64) if Cin % 64 == 0 else (32 if Cin % 32 == 0 else 16)
        if Cin % 64 == 0 and Cin % bn != 0 and Cin > bn:
            bn = 64
        base = -(-Cout // 128) * -(-Cin // bn) * k * k
        sp = max(1, min(-(-2 * sms // base), max(1, ksteps // 8)))
    per = -(-ksteps // sp)
    return kern, bn, -(-ksteps // per), ksteps % per != 0


# (B, H, W, Cin, Cout, k, stride, kernel, N tile, several slices); the split counts are those of a 132-SM H100
CASES = [
    (1, 8, 8, 128, 128, 1, 1, "general", 128, False),
    (4, 24, 23, 256, 192, 3, 1, "general", 128, True),       # Cout 192: a half-empty 128-row tile
    (2, 48, 40, 64, 128, 1, 1, "general", 64, True),
    (8, 128, 130, 64, 64, 1, 1, "general", 64, True),       # 260 slices of one tile, as on the 320 x 320 maps
    (4, 48, 44, 192, 64, 3, 2, "general", 64, True),          # Cin 192: three 64-wide tiles
    (2, 23, 21, 96, 64, 3, 1, "general", 32, True),           # K = 966: partial last k-step
    (3, 30, 30, 48, 64, 3, 2, "general", 16, False),
    (4, 40, 40, 16, 32, 3, 1, "general", 16, True),
    (2, 20, 20, 512, 255, 1, 1, "general", 128, False),       # the 255-wide head in a 256-channel buffer
    (8, 20, 20, 512, 255, 1, 1, "general", 128, True),
    (1, 9, 7, 32, 64, 3, 1, "taps", 64, False),
    (8, 40, 39, 32, 64, 3, 1, "taps", 64, True),
    (1, 8, 8, 64, 64, 3, 1, "taps", 32, False),
    (4, 40, 39, 64, 96, 3, 1, "taps", 32, True),
]
IDS = ["B%d_%dx%d_%d-%d_k%d_s%d" % c[:7] for c in CASES]


def make_case(case, seed=0, gdt=torch.float16):
    """operands (NHWC, dY possibly a channel slice of a wider buffer), a non-zero dW to accumulate into, and the fp64
    reference base + scale * dW."""
    B, H, W, Cin, Cout, k, stride = case[:7]
    pad = (k - 1) // 2
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g).to(gdt).double()
    w = torch.zeros(Cout, Cin, k, k, dtype=torch.double, requires_grad=True)
    y = F.conv2d(x, w, None, stride=stride, padding=pad)
    dy = torch.randn(y.shape, generator=g).to(gdt).double()
    y.backward(dy)
    scale = 0.375
    base = torch.randn(Cout, k, k, Cin, generator=g) * w.grad.pow(2).mean().sqrt().item() * scale
    ref = base.double() + scale * w.grad.permute(0, 2, 3, 1)
    xn = x.permute(0, 2, 3, 1).contiguous().to(gdt).cuda()
    wide = Cout if Cout % 8 == 0 else -(-Cout // 128) * 128
    dyb = torch.zeros(B, y.shape[2], y.shape[3], wide, dtype=gdt, device="cuda")
    dyb[..., :Cout] = dy.permute(0, 2, 3, 1).to(gdt).cuda()
    return xn, dyb[..., :Cout], base.cuda(), ref, scale


def run(ops, case, xn, dyn, base, scale):
    dw = base.clone()
    ops.conv2d_bwd_weight(xn, dyn, case[5], case[6], (case[5] - 1) // 2, scale=scale, dw=dw)
    return dw


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_wgrad_accumulates_into_prefilled_dw(case):
    ops = _ops()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kern, bn, splits, _ = plan(*case[:7], sms)
    assert (kern, bn) == case[7:9]
    if sms == 132:
        assert (splits > 1) == case[9], splits
    xn, dyn, base, ref, scale = make_case(case)
    dw = run(ops, case, xn, dyn, base, scale)
    again = run(ops, case, xn, dyn, base, scale)
    torch.cuda.synchronize()
    err = (dw.cpu().double() - ref).abs().max().item() / (ref - base.cpu().double()).pow(2).mean().sqrt().item()
    print("\n%s %s N%d splits %d: err/rms %.3g" % (case[:7], kern, bn, splits, err))
    assert err < 2e-4
    assert torch.equal(dw, again)


def test_wgrad_bf16_operands_and_device_scale():
    ops = _ops()
    case = (8, 40, 39, 32, 64, 3, 1)            # tap-transposed kernel, many slices
    xn, dyn, base, ref, scale = make_case(case, seed=3, gdt=torch.bfloat16)
    inv = torch.tensor([0.5], device="cuda")
    dw = base.clone()
    ops.conv2d_bwd_weight(xn, dyn, 3, 1, 1, scale=scale * 2, dw=dw, inv_scale=inv)
    torch.cuda.synchronize()
    err = (dw.cpu().double() - ref).abs().max().item() / (ref - base.cpu().double()).pow(2).mean().sqrt().item()
    assert err < 2e-4


def test_wgrad_two_streams_match_serial_bit_for_bit():
    """every case issued on two streams at once, three rounds, each stream running a different case at any time: each
    result equals the serial one bit for bit (the workspaces of the two streams never mix)."""
    ops = _ops()
    data = [(c,) + make_case(c, seed=i + 1) for i, c in enumerate(CASES)]
    serial = [run(ops, c, xn, dyn, base, sc) for c, xn, dyn, base, _, sc in data]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    main = torch.cuda.current_stream()
    for s in streams:
        s.wait_stream(main)
    outs = [[None] * len(data) for _ in range(3)]
    for rep in range(3):
        for i, (c, xn, dyn, base, _, sc) in enumerate(data):
            with torch.cuda.stream(streams[(rep + i) % 2]):
                outs[rep][i] = run(ops, c, xn, dyn, base, sc)
    torch.cuda.synchronize()
    for rep in range(3):
        for i in range(len(data)):
            assert torch.equal(outs[rep][i], serial[i]), (rep, CASES[i][:7])
