"""GPU: squeeze-excite forward / backward at batch sizes whose workspace sections are not 16-byte multiples.

The SE workspace holds [batch][c] means, pre-activations and gates and the [batch][cr] hidden activations; the gate
section is read with 16-byte loads.  With N * cr not a multiple of 4 (MobileNetV3: cr = c / 4 = 18, 30, ...; batch 1 or
3, e.g. a short last evaluation batch) the gate section must still start aligned."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers  # noqa: F401  (puts the package on sys.path)

pytestmark = pytest.mark.gpu


def _nhwc(t, dtype=torch.float16):
    return t.permute(0, 2, 3, 1).contiguous().to(dtype).cuda()


def _nchw(t):
    return t.float().permute(0, 3, 1, 2).cpu()


@pytest.mark.parametrize("B,C", [(1, 72), (3, 72), (3, 120), (5, 40)])
def test_squeeze_excite_odd_batch(B, C):
    from b200yolo import ops
    g = torch.Generator().manual_seed(B * 1000 + C)
    H, W = 6, 8
    cr = C // 4
    assert (B * cr) % 4 != 0
    x = (torch.randn(B, C, H, W, generator=g) + 0.5).half().float()
    w1 = torch.randn(cr, C, generator=g) / C ** 0.5 * 3
    w2 = torch.randn(C, cr, generator=g) / cr ** 0.5 * 3
    dy = torch.randn(B, C, H, W, generator=g).bfloat16().float()
    xr = x.clone().double().requires_grad_(True)
    w1r, w2r = w1.clone().double().requires_grad_(True), w2.clone().double().requires_grad_(True)
    pooled = xr.mean(dim=(2, 3))
    gate = F.relu6(F.relu(pooled @ w1r.t()) @ w2r.t() + 3.0) / 6.0
    ref = xr * gate.view(B, C, 1, 1)
    ref.backward(dy.double())
    xn = _nhwc(x)
    y, ws = ops.se_fwd(xn, w1.cuda(), w2.cuda())
    prev = torch.randn(B, C, H, W, generator=g).bfloat16()
    dx, dw1, dw2 = ops.se_bwd(xn, _nhwc(dy, torch.bfloat16), w1.cuda(), w2.cuda(), ws,
                              _nhwc(prev.float(), torch.bfloat16), accumulate=True, grad_scale=0.5)
    torch.cuda.synchronize()
    assert (_nchw(y) - ref.detach().float()).abs().max() < 2e-3 * max(1.0, float(ref.detach().abs().max()))
    want = prev.float() + xr.grad.float()
    assert (_nchw(dx) - want).abs().max() < 1.6e-2 * max(1.0, float(want.abs().max()))
    np.testing.assert_allclose(dw1.cpu().numpy() * 2, w1r.grad.float().numpy(), rtol=2e-3,
                               atol=2e-4 * float(w1r.grad.abs().max()))
    np.testing.assert_allclose(dw2.cpu().numpy() * 2, w2r.grad.float().numpy(), rtol=2e-3,
                               atol=2e-4 * float(w2r.grad.abs().max()))
