"""CPU: b200yolo.optim's parameter groups (train.py:120-144), tile table and flat state views."""
import numpy as np
import pytest
import torch

from helpers import build_model, cfg_path
from optim_ref import HYP, group_of, torch_optimizer

MODELS = [("yolov3-tiny", -1), ("yolov4", -1), ("yolov3-mobilenet", -1), ("yolov3-tiny", 1), ("yolov3-tiny", 2)]


def _model(name, quantized, seed=0):
    if quantized == -1:
        return build_model(name, seed=seed)
    import models
    torch.manual_seed(seed)
    return models.Darknet(cfg_path(name), quantized=quantized, a_bit=8, w_bit=8, shortcut_way=1, steps=100)


def _dp(name, quantized):
    from b200yolo.parallel import FlatDataParallel
    return FlatDataParallel(_model(name, quantized))


@pytest.mark.parametrize("name,quantized", MODELS)
def test_groups_follow_train_py(name, quantized):
    from b200yolo.optim import FlatAdam, FlatSGD, make_optimizer
    dp = _dp(name, quantized)
    names = {id(p): n for n, p in dp.module.named_parameters()}
    for adam in (False, True):
        opt = make_optimizer(dp, HYP, adam=adam, quantized=quantized)
        ref = torch_optimizer(dp.module, HYP, adam=adam, quantized=quantized)
        assert isinstance(opt, FlatAdam if (adam or quantized != -1) else FlatSGD)
        assert isinstance(opt, type(ref))
        assert len(opt.param_groups) == len(ref.param_groups) == (4 if quantized == 2 else 3)
        for g, r in zip(opt.param_groups, ref.param_groups):
            assert [names[id(p)] for p in g['params']] == [names[id(p)] for p in r['params']]
            assert {k: v for k, v in g.items() if k != 'params'} == {k: v for k, v in r.items() if k != 'params'}
        assert sum(len(g['params']) for g in opt.param_groups) == len(dp.params)
    order = ['pg0', 'pg3', 'pg1', 'pg2'] if quantized == 2 else ['pg0', 'pg1', 'pg2']
    for pg, g in zip(order, opt.param_groups):
        assert all(group_of(names[id(p)], quantized) == pg for p in g['params'])
    if quantized == 2:
        pg3 = [names[id(p)] for p in opt.param_groups[1]['params']]
        pg1 = [names[id(p)] for p in opt.param_groups[2]['params']]
        assert pg3 and all(n.endswith('activation_quantizer.scale') for n in pg3)
        assert any(n.endswith('Conv2d.weight_quantizer.scale') for n in pg1)        # the substring rule, literally


def _bn_idx(dp):
    return [i for i, m in enumerate(dp.module.module_list)
            if isinstance(m, torch.nn.Sequential) and len(m) > 1 and isinstance(m[1], torch.nn.BatchNorm2d)][::2]


@pytest.mark.parametrize("name,quantized", MODELS)
def test_tile_table_covers_each_element_once(name, quantized):
    from b200yolo import lib
    from b200yolo.optim import build_tile_table, make_optimizer
    dp = _dp(name, quantized)
    opt = make_optimizer(dp, HYP, quantized=quantized)
    l1_ids = set()
    if quantized == -1:
        idx = _bn_idx(dp)
        dp.set_bn_sparsity(idx, 1e-3)
        l1_ids = {id(dp.module.module_list[i][1].weight) for i in idx}
        assert l1_ids
    t = build_tile_table(dp, opt.param_groups).numpy()
    start, length, flags = t[:, 0], t[:, 1] & 0xffffffff, t[:, 1] >> 32
    n = dp.flat_param.numel()
    assert start[0] == 0 and np.all(start[1:] == start[:-1] + length[:-1]) and start[-1] + length[-1] == n
    assert np.all(length > 0) and np.all(length <= lib.OPT_TILE)
    bounds = np.cumsum([0] + [p.numel() for p in dp.params])
    owner = np.searchsorted(bounds, start, side='right') - 1
    assert np.array_equal(owner, np.searchsorted(bounds, start + length - 1, side='right') - 1)   # inside one tensor
    assert np.all((start == bounds[owner]) | (start % lib.OPT_TILE == 0))           # later tiles start 16-byte aligned
    group = {id(p): gi for gi, g in enumerate(opt.param_groups) for p in g['params']}
    want_g = np.array([group[id(dp.params[i])] for i in owner])
    want_l1 = np.array([id(dp.params[i]) in l1_ids for i in owner])
    assert np.array_equal(flags & 3, want_g)
    assert np.array_equal((flags & lib.OPT_TILE_L1) != 0, want_l1)


def _views_of(state_tensor, flat, off):
    return (state_tensor.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
            and state_tensor.storage_offset() == flat.storage_offset() + off)


@pytest.mark.parametrize("name,quantized,adam", [("yolov3-tiny", -1, False), ("yolov3-tiny", -1, True),
                                                 ("yolov3-tiny", 2, True)])
def test_state_is_views_of_flat_buffers_and_round_trips(name, quantized, adam):
    """A torch optimiser built by train.py's code, stepped twice on the CPU, loads into the flat optimiser as views of
    its flat buffers; the flat optimiser's state_dict loads back into a fresh torch optimiser unchanged."""
    from b200yolo.optim import make_optimizer
    dp = _dp(name, quantized)
    twin = _model(name, quantized, seed=1)
    ref = torch_optimizer(twin, HYP, adam=adam, quantized=quantized)
    g = torch.Generator().manual_seed(0)
    for _ in range(2):
        for p in twin.parameters():
            p.grad = torch.randn(p.shape, generator=g) * 1e-2
        ref.step()
    opt = make_optimizer(dp, HYP, adam=adam, quantized=quantized)
    sd = ref.state_dict()
    sd['param_groups'][0]['lr'] = 0.123
    opt.load_state_dict(sd)
    assert opt.param_groups[0]['lr'] == 0.123
    keys = ('exp_avg', 'exp_avg_sq') if (adam or quantized != -1) else ('momentum_buffer',)
    flats = {'momentum_buffer': dp.flat_mom}
    if 'exp_avg' in keys:
        flats = {'exp_avg': opt.exp_avg, 'exp_avg_sq': opt.exp_avg_sq}
    names = {id(p): n for n, p in dp.module.named_parameters()}
    twin_p = dict(twin.named_parameters())
    off = 0
    for p in dp.params:
        st = opt.state[p]
        for k in keys:
            assert _views_of(st[k], flats[k], off), (names[id(p)], k)
            assert torch.equal(st[k], ref.state[twin_p[names[id(p)]]][k])
        if 'exp_avg' in keys:
            assert float(st['step']) == 2.0
        off += p.numel()
    back = torch_optimizer(_model(name, quantized, seed=2), HYP, adam=adam, quantized=quantized)
    back.load_state_dict(opt.state_dict())
    got = back.state_dict()['state']
    assert got.keys() == sd['state'].keys()
    for i, b in sd['state'].items():
        assert got[i].keys() == b.keys() and all(torch.equal(got[i][k], b[k]) for k in b)
    assert back.param_groups[0]['lr'] == 0.123
    # zero_grad is one memset of the flat gradient; .grad stays the flat view
    dp.flat_grad.fill_(1.0)
    opt.zero_grad()
    assert not dp.flat_grad.any()
    assert all(p.grad is dp.grad_views[id(p)] for p in dp.params)
