"""GPU: plans of different input shapes share their device storage (b200yolo.engine.SlotStore).

Every comparison is against a private engine: a deepcopy of the model taken just before the step, whose engine owns a
single plan.  Multi-scale training and rectangular evaluation batches must compute exactly what those private plans
compute, whichever shapes ran before, while the storage grows, shrinks back to prefixes and is pinned by a pending
backward."""
import copy
import gc

import pytest
import torch

from helpers import attach_hyp, build_model, orc

pytestmark = pytest.mark.gpu

# visits every shape twice, growing the slots (64 -> 96 -> 128) and reading smaller prefixes of them afterwards
TRAIN_SHAPES = [(96, 96), (128, 128), (64, 64), (128, 96), (96, 128), (64, 64), (96, 96), (128, 96), (128, 128),
                (96, 128)]
EVAL_SHAPES = [(3, 96, 128), (3, 128, 96), (3, 128, 128), (1, 128, 128)]


def _targets(B):
    """Four targets per image, one per quadrant: never more than one target of an image in a grid cell at any of the
    shapes, so the loss-gradient scatter is deterministic."""
    rows = []
    for b in range(B):
        for j, (cx, cy) in enumerate([(0.3, 0.3), (0.7, 0.3), (0.3, 0.7), (0.7, 0.7)]):
            rows.append([b, (7 * b + 13 * j) % 80, cx + 0.01 * b, cy - 0.01 * j, 0.2 + 0.05 * j, 0.3 - 0.04 * j])
    return torch.tensor(rows, dtype=torch.float32)


def _step(model, x, t):
    """forward, compute_loss, backward; returns (p, loss items, {name: grad}, {name: buffer})."""
    from utils import utils as my_utils
    model.zero_grad(set_to_none=True)
    p, _ = model(x)
    loss, items = my_utils.compute_loss(p, t, model)
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: q.grad.detach().clone() for n, q in model.named_parameters() if q.grad is not None}
    bufs = {n: b.detach().clone() for n, b in model.named_buffers()}
    return [pi.detach().clone() for pi in p], items.detach().clone(), grads, bufs


def _private_step(model, x, t):
    priv = copy.deepcopy(model)
    out = _step(priv, x, t)
    del priv
    return out


def _assert_identical(got, ref, what):
    p, items, grads, bufs = got
    rp, ritems, rgrads, rbufs = ref
    for i, (a, b) in enumerate(zip(p, rp)):
        assert torch.equal(a, b), "%s: p[%d] differs from the private engine" % (what, i)
    rel = ((items - ritems).abs() / ritems.abs().clamp(min=1e-30)).max().item()
    assert rel <= 1e-6, "%s: loss items differ by %.3g (relative)" % (what, rel)
    assert grads.keys() == rgrads.keys()
    for n in grads:
        assert torch.equal(grads[n], rgrads[n]), "%s: gradient of %s differs" % (what, n)
    for n in bufs:
        assert torch.equal(bufs[n], rbufs[n]), "%s: buffer %s differs" % (what, n)


def _train_model(name):
    model = attach_hyp(build_model(name, device="cuda")).train()
    return model


@pytest.mark.parametrize("name", ["yolov3", "yolov4", "yolov3-mobilenet"])
def test_multiscale_training_bit_identical(name):
    model = _train_model(name)
    B = 2
    t = _targets(B).cuda()
    for k, (H, W) in enumerate(TRAIN_SHAPES):
        x = orc.synth_images(B, H, W, seed=k).cuda()
        ref = _private_step(model, x, t)
        got = _step(model, x, t)
        _assert_identical(got, ref, "%s step %d (%dx%d)" % (name, k, H, W))
    eng = model.engine()
    assert eng.train_store.generation > 0            # the sequence did grow the slots


@pytest.mark.parametrize("name", ["yolov3-tiny"])
def test_multiscale_training_with_atomics(name):
    """The overlapping 2x2 max-pool backward adds with 16-bit atomics, and batch-statistics BatchNorm over two small
    images amplifies the reordering: two private runs of the same step differ by up to ~10 % of a tensor's
    max.  Deviations are therefore taken relative to each tensor's max and compared as the worst over all outputs,
    gradients and running statistics of a step (the worst of many tensors is a stable yardstick; one small tensor is
    not): the shared run, against the closer private run, stays within twice the private spread plus 1e-3.  A wrong pad
    or a stale byte is far outside that."""
    model = _train_model(name)
    B = 2
    t = _targets(B).cuda()

    def worst(u, v):
        return max((a - b).abs().max().item() / max(b.abs().max().item(), 1e-30) for a, b in zip(u, v))

    def flat(r):
        return list(r[0]) + [r[2][n] for n in sorted(r[2])] + [r[3][n] for n in sorted(r[3])
                                                                  if r[3][n].is_floating_point()]

    for k, (H, W) in enumerate(TRAIN_SHAPES):
        x = orc.synth_images(B, H, W, seed=k).cuda()
        r1 = flat(_private_step(model, x, t))
        r2 = flat(_private_step(model, x, t))
        got = flat(_step(model, x, t))
        dev, spread = min(worst(got, r1), worst(got, r2)), worst(r1, r2)
        assert dev <= 2 * spread + 1e-3, "%s step %d (%dx%d): deviation %.3g, private spread %.3g" % (
            name, k, H, W, dev, spread)


def _eval_inputs(shape, dtype, seed):
    b, h, w = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (b, 3, h, w), dtype=torch.uint8, generator=g)
    return (x if dtype == torch.uint8 else x.float() / 256.0).cuda()


@pytest.mark.parametrize("name", ["yolov3-tiny", "yolov4", "yolov3-mobilenet"])
def test_rect_eval_bit_identical(name):
    """Bit for bit."""
    model = build_model(name, device="cuda").eval()
    batches = [(s, dt) for dt in (torch.uint8, torch.float32) for s in EVAL_SHAPES]

    def private(x):
        priv = copy.deepcopy(model)
        out = priv(x)
        del priv
        return [out[0]] + list(out[1])

    with torch.no_grad():
        for rnd in range(2):                        # the second round replays the cached plans' graphs
            for k, (shape, dt) in enumerate(batches):
                x = _eval_inputs(shape, dt, seed=10 * rnd + k)
                r1 = private(x)
                io, p, _ = model(x)
                got = [io] + list(p)
                what = "%s %s %s round %d" % (name, shape, dt, rnd)
                for i, (a, b) in enumerate(zip(got, r1)):
                    assert torch.equal(a, b), what + (": io differs" if i == 0 else ": p[%d] differs" % (i - 1))

        # static_outputs: each shape's returned buffers belong to its plan and survive forwards of the other shapes
        model.static_outputs = True
        kept = []
        for k, (shape, dt) in enumerate(batches):
            io, p, _ = model(_eval_inputs(shape, dt, seed=100 + k))
            kept.append((io, p, io.clone(), [q.clone() for q in p]))
        for k, (io, p, io_c, p_c) in enumerate(kept):
            assert torch.equal(io, io_c), "static io of batch %d was overwritten" % k
            for a, b in zip(p, p_c):
                assert torch.equal(a, b), "static p of batch %d was overwritten" % k


def _slot_bytes(store):
    return sum(s.numel() for s in store.slots.values())


def test_growth_frees_old_storage():
    model = _train_model("yolov3")
    B = 2
    t = _targets(B).cuda()
    eng = model.engine()
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    seen = {}
    for k, S in enumerate([64, 96, 128]):
        x = orc.synth_images(B, S, S, seed=k).cuda()
        for rep in range(2):                        # eager step, then the captured graphs
            ref = _private_step(model, x, t)
            got = _step(model, x, t)
            _assert_identical(got, ref, "growth %dx%d rep %d" % (S, S, rep))
        del ref, got, x
        model.zero_grad(set_to_none=True)
        gc.collect()
        torch.cuda.synchronize()
        # a grown slot drops every plan built on the old one: only the current shape stays cached
        assert len(eng.plans) == 1
        seen[S] = (torch.cuda.memory_allocated() - base, _slot_bytes(eng.train_store))
    alloc96, slots96 = seen[96]
    alloc128, slots128 = seen[128]
    assert slots96 > 16 * 2 ** 20
    assert slots128 > slots96
    # what is allocated besides the slots (weights, gradients, one plan's graphs) does not grow with the old storage
    assert alloc128 - slots128 <= (alloc96 - slots96) + 8 * 2 ** 20, (seen, "old slots were not freed")


def test_pin_forward_forward_backward_backward():
    from utils import utils as my_utils
    model = _train_model("yolov3")
    B = 2
    t = _targets(B).cuda()
    xa = orc.synth_images(B, 96, 96, seed=1).cuda()
    xb = orc.synth_images(B, 64, 64, seed=2).cuda()
    for x in (xa, xb, xa, xb):                      # both shapes cached, with their graphs
        _step(model, x, t)
    eng = model.engine()

    model.zero_grad(set_to_none=True)
    priv_a = copy.deepcopy(model)
    pa, _ = model(xa)
    la, _ = my_utils.compute_loss(pa, t, model)
    assert eng.train_store.pinned_by() is not None
    priv_b = copy.deepcopy(model)
    pb, _ = model(xb)
    assert eng.last_plan.store is not eng.train_store      # B runs on private storage while A waits
    lb, _ = my_utils.compute_loss(pb, t, model)
    lb.backward()
    gb = {n: q.grad.clone() for n, q in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    la.backward()
    ga = {n: q.grad.clone() for n, q in model.named_parameters()}
    assert eng.train_store.pinned_by() is None

    for priv, x, g, what in ((priv_a, xa, ga, "A"), (priv_b, xb, gb, "B")):
        ref = _step(priv, x, t)
        assert torch.equal(pa[0].detach() if what == "A" else pb[0].detach(), ref[0][0]), what + ": p differs"
        for n in g:
            assert torch.equal(g[n], ref[2][n]), "%s: gradient of %s differs" % (what, n)
    del priv_a, priv_b

    # after the backward has run, the next forward of the other shape is back on the shared storage
    model(xb)
    assert eng.last_plan.store is eng.train_store

    # a forward whose outputs and loss are dropped without a backward releases the pin as well
    pa, _ = model(xa)
    la, _ = my_utils.compute_loss(pa, t, model)
    assert eng.train_store.pinned_by() is eng.last_plan
    assert eng.plan_for(xb).store is not eng.train_store     # the private plan of a pinned step, not a cache lookup
    del pa, la
    gc.collect()
    assert eng.train_store.pinned_by() is None
    model(xb)
    assert eng.last_plan.store is eng.train_store


def test_cache_and_memory_eleven_sizes(monkeypatch):
    from b200yolo import train_engine
    monkeypatch.delenv("B2Y_MAX_PLANS", raising=False)
    counts = {"plans": 0, "graphs": 0}
    init = train_engine.TrainPlan.__init__
    capture = torch.cuda.CUDAGraph.capture_begin

    def counting_init(self, *a, **k):
        counts["plans"] += 1
        init(self, *a, **k)

    def counting_capture(self, *a, **k):
        counts["graphs"] += 1
        return capture(self, *a, **k)

    monkeypatch.setattr(train_engine.TrainPlan, "__init__", counting_init)
    monkeypatch.setattr(torch.cuda.CUDAGraph, "capture_begin", counting_capture)

    model = _train_model("yolov3-tiny")
    t = _targets(1).cuda()
    sizes = [32 * k for k in range(20, 9, -1)]      # 640 ... 320: the largest size sets the slot capacities
    yolo_bytes = {S: sum(3 * (S // s) ** 2 * 85 * 4 for s in (32, 16)) for S in sizes}
    grew = {}
    for cycle in range(2):
        before = dict(counts)
        for S in sizes:
            x = orc.synth_images(1, S, S, seed=S).cuda()
            gc.collect()
            torch.cuda.synchronize()
            m0 = torch.cuda.memory_allocated()
            for _ in range(2):                      # eager step, then the captured graphs
                _step(model, x, t)
            model.zero_grad(set_to_none=True)
            gc.collect()
            torch.cuda.synchronize()
            if cycle == 0:
                grew[S] = torch.cuda.memory_allocated() - m0
        if cycle == 1:
            assert counts == before, "second cycle built plans or captured graphs: %s -> %s" % (before, counts)
    assert len(model.engine().plans) == len(sizes)
    for S in sizes[1:]:
        assert grew[S] <= 4 * yolo_bytes[S] + 8 * 2 ** 20, (S, grew[S], yolo_bytes[S])
