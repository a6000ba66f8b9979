"""GPU: gradient-free train-mode forwards (adaptive BatchNorm recalibration, EagleEye_*_prune.py) on the forward-only
statistics plan: the logical-width BatchNorm kernel and the column-mapped weight pack, bit-identity with the training
forward on stock models, parity with the reference's recalibration of the pruned fixture models
(tests/golden/pruned_adabn_case.npz), the zero pad channels, a recalibration between a training forward and its backward,
and the flat data-parallel buffers."""
import copy

import pytest
import torch

from adabn_case import adabn_fixture, batches, eval_images, fixture_cases, oracle_recalibrate, rows, stat_keys
from helpers import attach_hyp, build_model, orc
from pruned_models import build_pruned, compact_defs

pytestmark = pytest.mark.gpu

CASES = [n for n, _ in fixture_cases()]
# batch statistics summed in a fixed order (double accumulators of the conv epilogues): the same batch, the same bits
STOCK = [("yolov3-tiny", 96), ("yolov3", 96), ("yolov4", 96), ("yolov2-tiny", 96)]
# gates of tests/test_gpu_train_model.py (train mode) and tests/test_gpu_pruned.py (eval)
POLICY_SLACK = 2.0
P_ABS_FLOOR = 0.02
STAT_TOL = 2e-2
BOX_REL_TOL_FP32REF = 3e-2
PROB_ABS_TOL_FP32REF = 1.5e-2
BOX_REL_TOL_EMU = 1e-2
PROB_ABS_TOL_EMU = 5e-3


def _bn_stats(model):
    return [(k, v.detach().clone()) for k, v in model.state_dict().items()
            if k.endswith(('running_mean', 'running_var', 'num_batches_tracked'))]


# ---- kernels ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["leaky", "mish", "linear"])
@pytest.mark.parametrize("residual", [False, True])
def test_bn_train_fwd_at_logical_width(act, residual):
    from b200yolo.lib import ACT, call, ptr, stream_ptr
    CL, CP, P = 37, 40, 4 * 13 * 11
    g = torch.Generator().manual_seed(3)
    z = torch.randn(P, CP, generator=g).half()
    z[:, CL:] = 0                                       # a conv with zero pad rows writes zero pad channels
    zf = z.float()
    s1, s2 = zf.sum(0).cuda(), (zf * zf).sum(0).cuda()
    z = z.cuda()
    res = torch.randn(P, CP, generator=g).half()
    res[:, CL:] = 0
    res = res.cuda() if residual else None
    CANARY = 1234.5
    gamma, beta = torch.rand(CL, generator=g) + 0.5, torch.randn(CL, generator=g)
    rm, rv = torch.randn(CL, generator=g), torch.rand(CL, generator=g) + 0.5

    def canaried(t):
        return torch.cat([t, torch.full((CP - CL,), CANARY)]).cuda()

    def padded(t, fill):
        return torch.cat([t, torch.full((CP - CL,), fill)]).cuda()

    lw = dict(gamma=canaried(gamma), beta=canaried(beta), rm=canaried(rm), rv=canaried(rv),
              save=torch.full((4, CP), CANARY).cuda(), y=torch.full((P, CP), 7.0).half().cuda())
    full = dict(gamma=padded(gamma, 0.0), beta=padded(beta, 0.0), rm=padded(rm, 0.0), rv=padded(rv, 1.0),
                save=torch.zeros(4, CP).cuda(), y=torch.zeros(P, CP).half().cuda())
    for entry, d in (("b2y_bn_train_fwd_lw", lw), ("b2y_bn_train_fwd", full)):
        args = [ptr(z), CP, ptr(s1), ptr(s2), P, ptr(d['gamma']), ptr(d['beta']), 1e-5, 0.1, ptr(d['rm']), ptr(d['rv']),
                ptr(d['save']), ptr(res), CP if residual else 0, ptr(d['y']), CP, P, CP]
        args += [CL] if entry.endswith("_lw") else []
        call(entry, *args, ACT[act], 0.1, stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(lw['y'][:, :CL], full['y'][:, :CL])
    assert torch.equal(lw['y'][:, CL:], torch.zeros_like(lw['y'][:, CL:]))
    assert torch.equal(lw['rm'][:CL], full['rm'][:CL]) and torch.equal(lw['rv'][:CL], full['rv'][:CL])
    assert torch.equal(lw['save'][:, :CL], full['save'][:, :CL])
    for k in ('gamma', 'beta', 'rm', 'rv'):
        assert torch.equal(lw[k][CL:], torch.full((CP - CL,), CANARY, device='cuda')), k
    assert torch.equal(lw['save'][:, CL:], torch.full((4, CP - CL), CANARY, device='cuda'))


@pytest.mark.parametrize("k,stride", [(3, 1), (3, 2), (1, 1)])
def test_pack_with_column_map_equals_identity_pack_of_scattered_weights(k, stride):
    from b200yolo.lib import PackItem, call, ptr, raw, stream_ptr
    O, Opad, I = 37, 40, 37
    cmap = list(range(21)) + list(range(24, 40))         # [21 | 16]: a concat of two pruned widths, gap at 21..23
    Ipad = 48
    g = torch.Generator().manual_seed(5)
    w = torch.randn(O, I, k, k, generator=g).cuda()
    ws = torch.zeros(O, Ipad, k, k, device='cuda')
    ws[:, cmap] = w
    cm = torch.tensor(cmap, dtype=torch.int32, device='cuda')
    ti = int(raw().b2y_layout_tile_i(k))
    outs = []
    for src, n_in, colmap in ((w, I, cm), (ws, Ipad, None)):
        wf = torch.zeros(Opad, k, k, Ipad, dtype=torch.float16, device='cuda')
        it = PackItem(src.data_ptr(), wf.data_ptr(), None, O, Opad, n_in, k, stride, k // 2, 0, Ipad,
                      colmap.data_ptr() if colmap is not None else None)
        tab = torch.frombuffer(bytearray(bytes((PackItem * 1)(it))), dtype=torch.uint8).cuda()
        call("b2y_pack_conv_weights_multi", ptr(tab), 1, ((Opad + 31) // 32) * ((n_in + ti - 1) // ti), stream_ptr())
        outs.append(wf)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0][..., 21:24], torch.zeros_like(outs[0][..., 21:24]))
    assert torch.equal(outs[0][O:], torch.zeros_like(outs[0][O:]))


# ---- stock models: the same numbers as the training forward ------------------------------------------------------------
@pytest.mark.parametrize("name,S", STOCK)
@pytest.mark.parametrize("graph", [True, False])
def test_stock_gradient_free_forward_is_the_training_forward(name, S, graph):
    ref = build_model(name, device="cuda").train()
    mine = copy.deepcopy(ref)
    for m in (ref, mine):
        m.use_cuda_graph = graph
    for step in range(3):                               # eager, capture, replay
        x = orc.synth_images(2, S, S, seed=40 + step).cuda()
        p_ref, _ = ref(x)
        assert p_ref[0].requires_grad
        with torch.no_grad():
            p_mine, _ = mine(x)
        torch.cuda.synchronize()
        assert type(mine.engine().last_plan) is type(ref.engine().last_plan)
        assert mine.engine().last_plan.forward_only and not ref.engine().last_plan.forward_only
        for a, b in zip(p_mine, p_ref):
            assert torch.equal(a, b.detach()), (name, step)
        for (k, a), (_, b) in zip(_bn_stats(mine), _bn_stats(ref)):
            assert torch.equal(a, b), (name, step, k)
        del p_ref


def test_stock_mobilenet_gradient_free_forward_within_atomics_reordering():
    """The gradient-free forward of stock MobileNet stays within three times the spread of two training forwards of the
    same batch, relative to each tensor's max, plus 1e-3."""
    ref = build_model("yolov3-mobilenet", device="cuda").train()
    ref2, mine = copy.deepcopy(ref), copy.deepcopy(ref)

    def worst(u, v):
        return max((a - b).abs().max().item() / max(b.abs().max().item(), 1e-30) for a, b in zip(u, v))
    for step in range(3):                               # eager, capture, replay
        x = orc.synth_images(2, 128, 128, seed=40 + step).cuda()
        p_ref, _ = ref(x)
        p_ref2, _ = ref2(x)
        with torch.no_grad():
            p_mine, _ = mine(x)
        torch.cuda.synchronize()
        assert mine.engine().last_plan.forward_only
        r = [t.detach() for t in p_ref] + [v for k, v in _bn_stats(ref) if v.is_floating_point()]
        r2 = [t.detach() for t in p_ref2] + [v for k, v in _bn_stats(ref2) if v.is_floating_point()]
        m = list(p_mine) + [v for k, v in _bn_stats(mine) if v.is_floating_point()]
        assert worst(m, r) <= 3 * worst(r2, r) + 1e-3, (step, worst(m, r), worst(r2, r))
        assert all(torch.equal(a, b) for (k, a), (_, b) in zip(_bn_stats(mine), _bn_stats(ref))
                   if k.endswith('num_batches_tracked'))
        del p_ref, p_ref2


def test_frozen_parameters_take_the_forward_only_plan():
    model = build_pruned("yolov3-tiny", device="cuda").train()
    for p in model.parameters():
        p.requires_grad_(False)
    p, _ = model(batches("yolov3-tiny")[0].cuda())     # grad mode on, nothing to differentiate
    assert model.engine().last_plan.forward_only and not p[0].requires_grad


def test_growing_batch_reuses_the_pack_table_safely():
    """A larger batch grows the forward-only slots, which drops the smaller batch's plan; the new plan reuses the pack
    table cached with the model's shared state, whose column maps must still be alive.  The gapped concat of the pruned
    yolov3-tiny (route 20) needs one.  The graphed model, after other allocations have taken over freed blocks (zero
    filled), computes what an eager fresh model computes on the same batches."""
    xs = [batches("yolov3-tiny")[0][:2], batches("yolov3-tiny")[1]]
    seq = [0, 1, 1, 1, 1]                               # B = 2, then B = 4: eager, capture, replay, replay
    graphed = build_pruned("yolov3-tiny", device="cuda").train()
    eager = build_pruned("yolov3-tiny", device="cuda").train()
    eager.use_cuda_graph = False
    filler = []
    with torch.no_grad():
        for k, j in enumerate(seq):
            p_g, _ = graphed(xs[j].cuda())
            p_e, _ = eager(xs[j].cuda())
            if k == 1:
                assert graphed.engine().train_store.generation > 0      # the slots grew
                filler = [torch.zeros(n, dtype=torch.int32, device="cuda") for n in range(1, 512) for _ in range(4)]
            torch.cuda.synchronize()
            for a, b in zip(p_g, p_e):
                assert torch.equal(a, b), k
    for (key, a), (_, b) in zip(_bn_stats(graphed), _bn_stats(eager)):
        assert torch.equal(a, b), key
    del filler


# ---- pruned models against the reference --------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_pruned_recalibration_matches_reference(name):
    g = adabn_fixture()
    model = build_pruned(name, device="cuda").train()
    epoch0 = getattr(model, '_b2y_epoch', 0)
    # yardstick: the oracle under the engine's precision policy
    emu_state = {k: v.cpu().clone() for k, v in model.state_dict().items()}
    p_emu = oracle_recalibrate(name, emu_state, emulate_fp16=True)
    mine_p = yard_p = 0.0
    for b, x in enumerate(batches(name)):
        with torch.no_grad():
            p, feats = model(x.cuda())
        for j, pj in enumerate(p):
            ref = torch.from_numpy(g["%s:p%d_%d" % (name, b, j)])
            assert pj.dtype == torch.float32 and pj.shape[-1] == ref.shape[-1]
            mine_p = max(mine_p, (rows(pj.cpu()) - ref).abs().max().item())
            yard_p = max(yard_p, (rows(p_emu[b][j]) - ref).abs().max().item())
    assert model._b2y_epoch > epoch0
    sd = model.state_dict()
    stat_err = yard_stat = 0.0
    for k in stat_keys(name):
        ref = torch.from_numpy(g["%s:stat::%s" % (name, k)])
        if k.endswith('num_batches_tracked'):
            assert int(sd[k]) == int(ref) == 3, k
            continue
        scale = ref.abs().clamp(min=1.0)
        stat_err = max(stat_err, ((sd[k].cpu() - ref).abs() / scale).max().item())
        yard_stat = max(yard_stat, ((emu_state[k] - ref).abs() / scale).max().item())
    # eval after the recalibration: the engine's own statistics through the eval plan, and against the reference
    model.eval()
    x = eval_images(name)
    with torch.no_grad():
        io = model(x.cuda())[0].cpu()
        io_emu, _ = orc.darknet_forward(compact_defs(name)[1:], {k: v.cpu() for k, v in sd.items()}, x, name,
                                        emulate_fp16=True)
    io, io_emu, io_ref = rows(io), rows(io_emu), torch.from_numpy(g[name + ":io"])

    def errs(got, want):
        return (((got[..., :4] - want[..., :4]).abs() / want[..., :4].abs().clamp(min=1.0)).max().item(),
                (got[..., 4:] - want[..., 4:]).abs().max().item())
    be, pe = errs(io, io_emu)
    bf, pf = errs(io, io_ref)
    print("\n[adabn %s] max|dp| %.3g (policy yardstick %.3g) | running stats rel %.3g (yardstick %.3g) | eval vs "
          "fp16-policy oracle box %.3g prob %.3g | vs reference box %.3g prob %.3g"
          % (name, mine_p, yard_p, stat_err, yard_stat, be, pe, bf, pf))
    assert mine_p <= POLICY_SLACK * yard_p + P_ABS_FLOOR
    assert stat_err < max(STAT_TOL, POLICY_SLACK * yard_stat)
    assert be <= BOX_REL_TOL_EMU and pe <= PROB_ABS_TOL_EMU
    assert bf <= BOX_REL_TOL_FP32REF and pf <= PROB_ABS_TOL_FP32REF


@pytest.mark.parametrize("name", CASES)
def test_pruned_feature_out_has_logical_widths(name):
    from b200yolo.layout import feature_slots
    model = build_pruned(name, device="cuda").train()
    model.keep_features = True
    with torch.no_grad():
        _, feats = model(batches(name)[0].cuda())
        got = [feats[j].cpu() for j in range(len(feats))]
    shapes = model.engine().last_plan.layout.shapes
    slots = feature_slots(model)
    assert len(got) == len(slots)
    for f, i in zip(got, slots):
        assert tuple(f.shape[1:]) == tuple(shapes[i]) and torch.isfinite(f).all(), i


@pytest.mark.parametrize("name", CASES)
def test_pad_and_gap_channels_stay_zero(name):
    model = build_pruned(name, device="cuda").train()
    model.use_cuda_graph = False
    with torch.no_grad():
        model(batches(name)[0].cuda())
    torch.cuda.synchronize()
    plan = model.engine().last_plan
    lay = plan.layout
    checked = 0
    for i, t in enumerate(lay.tens):
        if t is None or t.dtype != torch.float16 or t.buf is None:
            continue
        phys = t.buf[..., t.c0:t.c0 + t.Cp]
        pad = sorted(set(range(t.Cp)) - set(lay.chmap[i]))
        if pad:
            assert torch.count_nonzero(phys[..., pad]).item() == 0, (name, i)
            checked += 1
    assert checked


# ---- a recalibration between a training forward and its backward -----------------------------------------------------
def test_interleaved_recalibration_keeps_the_step():
    from utils import utils as my_utils
    x = orc.synth_images(4, 128, 128, seed=0).cuda()
    x2 = orc.synth_images(4, 128, 128, seed=1).cuda()
    t = orc.synth_targets(4, 6, 80, seed=1).cuda()

    def steps(interleave):
        model = attach_hyp(build_model("yolov3-tiny", device="cuda")).train()
        out = []
        for _ in range(3):                              # eager, capture, replay
            model.zero_grad(set_to_none=True)
            pred, _ = model(x)
            loss, _ = my_utils.compute_loss(pred, t, model)
            if interleave:
                # everything the step saved for its backward: the training plan's slots and BatchNorm statistics
                plan = model.engine().last_plan
                saved = {n: v.clone() for n, v in plan.store.slots.items() if n[0] != 'fo'}
                saved.update({('save', r.i): r.save.clone() for r in plan.convs if r.save is not None})
                with torch.no_grad():
                    model(x2)                           # same model and shape, between the forward and the backward
                assert model.engine().last_plan.forward_only
                torch.cuda.synchronize()
                for n, v in saved.items():
                    cur = plan.store.slots[n] if n[0] != 'save' else next(r.save for r in plan.convs if r.i == n[1])
                    assert torch.equal(cur, v), n
            loss.backward()
            out.append((float(loss), {k: p.grad.clone() for k, p in model.named_parameters()}))
        return out

    a, a2, b = steps(False), steps(False), steps(True)

    def worst(u, v):
        return max(float((u[1][k] - v[1][k]).norm() / (u[1][k].norm() + 1e-12)) for k in u[1])
    # two runs of the same step differ by the reordering of the loss and gradient atomics (tests/test_gpu_train_model.py)
    for s in range(3):
        noise = worst(a[s], a2[s])
        assert abs(a[s][0] - b[s][0]) <= max(1e-5 * abs(a[s][0]), 3 * abs(a[s][0] - a2[s][0]))
        assert worst(a[s], b[s]) < max(5e-2, 3 * noise), (s, worst(a[s], b[s]), noise)


# ---- flat data-parallel buffers ----------------------------------------------------------------------------------------
def test_recalibration_updates_the_flat_buffers_in_place():
    from b200yolo.parallel import FlatDataParallel
    plain = build_pruned("yolov3-tiny", device="cuda").train()
    wrapped = build_pruned("yolov3-tiny", device="cuda").train()
    dp = FlatDataParallel(wrapped)
    before = dp.flat_buf.clone()
    with torch.no_grad():
        for x in batches("yolov3-tiny"):
            plain(x.cuda())
            dp(x.cuda())
    torch.cuda.synchronize()
    assert not torch.equal(before, dp.flat_buf)
    lo, hi = dp.flat_buf.data_ptr(), dp.flat_buf.data_ptr() + dp.flat_buf.numel() * 4
    for (k, a), (_, b) in zip(_bn_stats(wrapped), _bn_stats(plain)):
        if a.dtype.is_floating_point:
            assert lo <= dict(wrapped.named_buffers())[k].data_ptr() < hi, k
        assert torch.equal(a, b), k
