"""CPU: the forward-only statistics plan (gradient-free train-mode forwards, adaptive BatchNorm recalibration of
channel-pruned models) is built on the CPU for every pruned fixture model: buffers at the physical widths, no backward
state; and the oracle reproduces the reference's recalibration (tests/golden/pruned_adabn_case.npz)."""
import pytest
import torch

from adabn_case import adabn_fixture, fixture_cases, oracle_recalibrate, rows, stat_keys
from pruned_models import build_pruned

CASES = [n for n, _ in fixture_cases()]


def _fo_plan(model, S, keep, store=None, shared=None):
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainPlan, TrainShared
    dev = torch.device("cpu")
    return TrainPlan(model, (2, 3, S, S), dev, keep, store or SlotStore(dev), shared or TrainShared(dev),
                     forward_only=True)


def _bound_tensors(plan):
    """(kind, fp16 tensor) of every tensor a forward step reads or writes"""
    from b200yolo.layout import _Tensor
    for st in plan.order:
        if st[0] in ('conv', 'se') and len(st) == 2:
            fields = [getattr(st[1], a, None) for a in ('src', 'y', 'z', 'res')]
        else:
            fields = list(st)
        for f in fields:
            if isinstance(f, _Tensor) and f.dtype == torch.float16:
                yield st[0], f


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("keep", [False, True])
def test_forward_only_plan_binds_physical_widths(name, keep):
    S = dict(fixture_cases())[name]
    model = build_pruned(name)
    plan = _fo_plan(model, S, keep)
    seen = 0
    for kind, f in _bound_tensors(plan):
        v = f.view()
        assert v.shape[3] == f.Cp and f.Cp % 8 == 0 and f.c0 % 8 == 0 and f.c0 + f.Cp <= f.buf.shape[3], (kind, f.C)
        seen += f.C != f.Cp
    assert seen, "the fixture has pruned widths"
    for r in plan.convs:
        if r.src is not None:
            # the forward GEMM reads the source up to its MMA K granule, inside the buffer; the packed weights are as wide
            if not r.depthwise:
                assert r.src.view_k().shape[3] == r.Ipad == r.w16.shape[3] and r.w16.shape[0] >= r.y.Cp
        if r.bn is not None:
            assert r.z.view().shape[3] == r.y.Cp and tuple(r.stats.shape) == (2, r.y.Cp)
            assert tuple(r.save.shape) == (4, r.y.Cp)
        if r.depthwise:
            assert r.wdw.shape[0] == r.src.Cp
    # every layer whose input a concat placed with gaps packs its weight columns through the channel map
    lay = plan.layout
    for r in plan.convs:
        if r.src is not None and not r.depthwise:
            ident = lay.chmap[r.i - 1] == tuple(range(r.conv.in_channels))
            assert (r.col_map is None) == ident
            if not ident:
                assert r.col_map.tolist() == list(lay.chmap[r.i - 1])


@pytest.mark.parametrize("name", CASES)
def test_forward_only_plan_holds_no_backward_state(name):
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainShared
    dev = torch.device("cpu")
    S = dict(fixture_cases())[name]
    store, shared = SlotStore(dev), TrainShared(dev)
    plan = _fo_plan(build_pruned(name), S, False, store, shared)
    for attr in ('bwd_arena', 'dz_bufs', 'dz_aux', 'grad_of', 'first_write'):
        assert getattr(plan, attr, None) in (None, {}), attr
    assert all(r.wT is None and r.dw is None and r.dwg is None and r.sums is None for r in plan.convs)
    assert not shared.wT and all(k[0] == 'fo' for k in shared.w16)
    # its slots are its own: nothing a training step saves for its backward is named like them
    assert store.slots and all(n[0] == 'fo' for n in store.slots)
    assert not any(n[1][0] in ('dz', 'bwd_arena', 'se_ws_bwd') for n in store.slots)
    # one z slot serves every BatchNorm layer
    assert sum(n[1][0] == 'z' for n in store.slots) == 1


def test_grad_enabled_constructor_still_refuses_pruned_widths():
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainPlan, TrainShared
    dev = torch.device("cpu")
    for name, S in fixture_cases():
        with pytest.raises(NotImplementedError, match=r"layer \d+: BatchNorm training needs a multiple of 8"):
            TrainPlan(build_pruned(name), (2, 3, S, S), dev, False, SlotStore(dev), TrainShared(dev))


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_recalibration(name):
    g = adabn_fixture()
    model = build_pruned(name)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    threads = torch.get_num_threads()
    torch.set_num_threads(1)          # CPU reductions in the generator's order
    try:
        ps = oracle_recalibrate(name, state)
    finally:
        torch.set_num_threads(threads)
    for b, p in enumerate(ps):
        for j, pj in enumerate(p):
            ref = torch.from_numpy(g["%s:p%d_%d" % (name, b, j)])
            assert ((rows(pj) - ref).abs().max() / ref.abs().max()).item() < 1e-5, (b, j)
    keys = stat_keys(name)
    assert keys and sum(k.endswith('running_mean') for k in keys) == sum(
        isinstance(m, torch.nn.BatchNorm2d) for m in model.modules())
    for k in keys:
        ref = torch.from_numpy(g["%s:stat::%s" % (name, k)])
        if k.endswith('num_batches_tracked'):
            assert int(ref) == len(ps)
            continue
        err = ((state[k] - ref).abs() / ref.abs().clamp(min=1e-3)).max().item()
        assert err < 1e-5, (k, err)


def test_pack_table_column_maps_outlive_the_plans():
    """The forward-only pack table is cached in TrainShared, keyed by the weight pointers, and holds the device pointers
    of the input-column maps: the maps live in TrainShared too, so a plan of another shape that reuses the table after
    the first plan was dropped never points at freed memory."""
    from b200yolo.engine import SlotStore
    from b200yolo.train_engine import TrainPlan, TrainShared
    dev = torch.device("cpu")
    store, shared = SlotStore(dev), TrainShared(dev)
    model = build_pruned("yolov3-tiny")
    small = TrainPlan(model, (2, 3, 96, 96), dev, False, store, shared, forward_only=True)
    maps = {r.i: r.col_map for r in small.convs if r.col_map is not None}
    assert maps, "the fixture has a gapped concat"
    del small
    large = TrainPlan(model, (4, 3, 96, 96), dev, False, store, shared, forward_only=True)
    for r in large.convs:
        if r.col_map is not None:
            assert r.col_map is maps[r.i]
    assert all(any(m is v for v in shared.col_maps.values()) for m in maps.values())
