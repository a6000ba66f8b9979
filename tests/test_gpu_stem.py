"""GPU: every first layer the plans can be given, in_c = 1..4, k = 1..7, stride 1 and 2, end to end through the
engine: an eval forward, a gradient-free train-mode forward and one training step of a one-conv-plus-head model
against fp64 torch, on whichever path layout.stem_path picks.  A shape is either computed or refused when its plan is
built; none may fail in a launch."""
import pytest
import torch
import torch.nn.functional as F

from helpers import stem_model

pytestmark = pytest.mark.gpu

B, H, W = 2, 40, 48
# the stem's output rounded to fp16 after an fp32 sum of fp16 (tensor-core paths) or fp32 (direct) operands
FWD_TOL = 2e-3
# The weight gradient of one step sums a product dz * x per output pixel.  Its error is measured per weight against
# the root-sum-square of those products (dz at fixed batch statistics), not against the gradient itself: the BatchNorm
# backward takes out of dz its components along the batch mean and along z, so that with few taps the sum nearly
# cancels (one tap: BatchNorm makes the loss invariant to the weight's scale, the gradient is ~0).  The gradient that
# reaches the stem through the head's bf16 data gradient is itself a few per cent off fp64 per element (its channel
# sums, the BatchNorm bias gradient, by up to 3 %), which bounds what the stem can reach: 0.14 at worst on this grid.
DW_TOL = 0.25

SHAPES = [(c, k, s) for c in range(1, 5) for k in range(1, 8) for s in (1, 2)]


def _half(t, tc):
    return t.half().double() if tc else t


def _ref_eval(m, x, tc):
    """fp64 eval forward of the stem: BatchNorm folded into the weights, as the plan packs them."""
    conv, bn = m.module_list[0].Conv2d, m.module_list[0].BatchNorm2d
    scale = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    wf = conv.weight.double() * scale.view(-1, 1, 1, 1)
    bf = bn.bias.double() - bn.running_mean.double() * scale
    z = F.conv2d(_half(x, tc), _half(wf, tc), bf, stride=conv.stride, padding=conv.padding)
    return F.leaky_relu(z, 0.1)


def _ref_train(m, x, tc, R=None):
    """fp64 train-mode forward (batch statistics) and, given R, the stem's weight gradient of sum(p * R) with the
    root-sum-square of its per-pixel terms, dz taken at fixed batch statistics."""
    conv, bn, head = m.module_list[0].Conv2d, m.module_list[0].BatchNorm2d, m.module_list[1].Conv2d
    yolo = m.module_list[2]
    w = conv.weight.detach().double().requires_grad_(True)
    xs = _half(x, tc)
    z = F.conv2d(xs, w if R is not None else _half(w, tc), None, stride=conv.stride, padding=conv.padding)

    def rest(z, stats):
        y = F.leaky_relu(F.batch_norm(z, *stats, bn.weight.double(), bn.bias.double(), stats == (None, None), 0.0,
                                      bn.eps), 0.1)
        p = F.conv2d(y, head.weight.double(), head.bias.double())
        return y, p.view(B, yolo.na, yolo.no, p.shape[2], p.shape[3]).permute(0, 1, 3, 4, 2)

    y, p = rest(z, (None, None))
    if R is None:
        return y, None, None
    (p * R).sum().backward()
    zf = z.detach().requires_grad_(True)
    (rest(zf, (zf.mean((0, 2, 3)).detach(), zf.var((0, 2, 3), unbiased=False).detach()))[1] * R).sum().backward()
    rss = torch.nn.grad.conv2d_weight(xs * xs, w.shape, zf.grad * zf.grad, conv.stride, conv.padding).sqrt()
    return y, w.grad, rss


def _check_fwd(got, ref, tag):
    err = (got.double() - ref).abs().max().item()
    assert got.shape == ref.shape and err <= FWD_TOL * max(1.0, ref.abs().max().item()), (tag, err)


@pytest.mark.parametrize("in_c,k,stride", SHAPES)
def test_first_layer_shape(in_c, k, stride):
    from b200yolo.layout import STEM_WGRAD_MAX_TAPS, stem_path
    filters = 32 if stride == 1 else 72          # wider than the fused kernel's 64 outputs: the eval im2col GEMM
    model = stem_model(in_c, k, stride, filters=filters, seed=in_c * 100 + k * 10 + stride)
    model.keep_features = True
    model.use_cuda_graph = False
    cpu = {n: t.detach().clone() for n, t in model.state_dict().items()}
    ref_model = stem_model(in_c, k, stride, filters=filters)
    ref_model.load_state_dict(cpu)
    model = model.cuda()
    g = torch.Generator().manual_seed(k * 10 + in_c)
    x = torch.rand(B, in_c, H, W, generator=g) * 2 - 1
    x64 = x.double()

    with torch.no_grad():
        ref_model.eval()
        eval_path = stem_path(in_c, k, filters)
        _, _, feats = model.eval()(x.cuda())
        _check_fwd(feats[0].cpu(), _ref_eval(ref_model, x64, eval_path != 'direct'), ("eval", eval_path))
        assert model.engine().last_plan.stem == eval_path

        train_path = stem_path(in_c, k, filters, training=True)
        _, feats = model.train()(x.cuda())
        assert model.engine().last_plan.convs[0].stem == train_path
        y_ref = _ref_train(ref_model, x64, train_path != 'direct')[0]
        _check_fwd(feats[0].cpu(), y_ref, ("train forward", train_path))

    R = torch.randn(B, 3, *feats[0].shape[2:], 6, generator=g)
    model.zero_grad()
    if train_path == 'direct' and in_c * k * k > STEM_WGRAD_MAX_TAPS:
        with pytest.raises(NotImplementedError, match="layer 0: the weight gradient"):
            model(x.cuda())
        return
    pred, feats = model(x.cuda())
    _check_fwd(feats[0].cpu(), y_ref, ("training step forward", train_path))
    (pred[0] * R.cuda()).sum().backward()
    torch.cuda.synchronize()
    _, dw_ref, rss = _ref_train(ref_model, x64, train_path != 'direct', R.double())
    dw = model.module_list[0].Conv2d.weight.grad.cpu().double()
    err = ((dw - dw_ref).abs() / rss).max().item()
    print("\n%s: weight gradient error %.3g of the root-sum-square of its terms" % ((in_c, k, stride, train_path), err))
    assert err <= DW_TOL, (train_path, err)
