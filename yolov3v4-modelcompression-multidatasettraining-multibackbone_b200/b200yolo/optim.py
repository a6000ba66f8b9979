"""train.py's optimiser over FlatDataParallel's flat buffers: per-group Nesterov SGD or Adam in ONE launch per step.

Reference: train.py:120-150 (parameter groups pg0 "other", [pg3 TPSQ scales], pg1 'Conv2d.weight' with weight decay,
pg2 '.bias'; Adam for --adam and for every QAT run, SGD-Nesterov otherwise), :356-365 (burn-in edits lr, weight_decay
and, when present, momentum of each group), :450-459 (optimizer.step / zero_grad), :549-573 (optimizer.state_dict in
the checkpoint).

FlatSGD and FlatAdam are torch.optim.SGD / torch.optim.Adam subclasses, so their param_groups carry torch's keys and
the burn-in loop, LambdaLR and MultiStepLR work on them unchanged.  step() reads every group's current values on the
host, packs them into a struct passed to the kernel by value, and launches csrc/train.cu opt_grouped_kernel once over a
device-resident tile table (built on the first step, rebuilt only when the groups or the BatchNorm-L1 set change).  The
gradient scale 1/world, the BatchNorm-L1 term (FlatDataParallel.set_bn_sparsity) and the model EMA
(FlatDataParallel.enable_ema) are applied in the same pass.  FlatDataParallel.step is a FlatSGD step over two groups.

Per-parameter state ('momentum_buffer', 'exp_avg', 'exp_avg_sq') are views of flat state buffers in the parameter
layout; state_dict() returns copies that load into a torch.optim.SGD / Adam built by train.py's code, and
load_state_dict() copies a torch optimiser's state into the flat views.  FlatSGD keeps its momentum in
FlatDataParallel.flat_mom, and whether that holds one in FlatDataParallel.has_momentum, so FlatDataParallel.step and
every FlatSGD over the same FlatDataParallel continue one momentum.
"""
from collections import defaultdict

import torch

from . import lib, ops
from .parallel import _is_decay_param


def train_param_groups(dp, quantized=-1):
    """train.py:125-133 over dp's parameters, in model.named_parameters() order: returns (pg0, pg1, pg2, pg3), pg3 None
    unless quantized == 2.  The substring rule is applied literally, so TPSQ's 'Conv2d.weight_quantizer.scale' lands in
    pg1 as it does in the reference."""
    flat = {id(p) for p in dp.params}
    pg0, pg1, pg2, pg3 = [], [], [], []
    for k, v in dict(dp.module.named_parameters()).items():
        if id(v) not in flat:
            raise ValueError("parameter %s is not in the FlatDataParallel buffers (requires_grad=False?)" % k)
        if _is_decay_param(k):
            pg1.append(v)
        elif '.bias' in k:
            pg2.append(v)
        elif 'scale' in k and quantized == 2:
            pg3.append(v)
        else:
            pg0.append(v)
    return pg0, pg1, pg2, (pg3 if quantized == 2 else None)


class _FlatOptimizer:
    """The flat-buffer machinery shared by FlatSGD and FlatAdam (placed before the torch class in the MRO)."""

    def _flat_init(self, dp):
        self.dp = dp
        self._tiles = None
        self._tiles_l1 = None

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        self._tiles = None

    def _tile_table(self):
        """int64 [n][2] device table of B2YOptTile rows {start, len | flags << 32}: tiles of at most OPT_TILE elements
        inside one parameter tensor, cut at multiples of OPT_TILE so that every tile but a tensor's first starts
        16-byte aligned."""
        l1 = self.dp._l1
        if self._tiles is not None and self._tiles_l1 is l1:
            return self._tiles
        self._tiles = build_tile_table(self.dp, self.param_groups)
        self._tiles_l1 = l1
        return self._tiles

    def _step_common(self):
        """The fields of lib.OptStep that do not depend on the algorithm; advances the EMA counter."""
        dp = self.dp
        hp = lib.OptStep()
        gs = 1.0 / float(dp.world)
        hp.grad_scale = gs
        if dp._l1 is not None:
            hp.l1_coeff = dp._l1[1] / gs          # updateBN runs on the averaged gradient, the kernel scales after it
        ema = getattr(dp, 'ema_param', None)
        d = 0.0
        if ema is not None:
            dp.ema_updates += 1
            d = dp._ema_decay(dp.ema_updates)
        hp.ema_decay = d
        return hp, ema, d

    def _step_done(self, ema, d):
        dp = self.dp
        if ema is not None and dp.ema_buf is not None:
            ops.axpby(dp.flat_buf, dp.ema_buf, 1.0 - d, d)          # running statistics: ema = d*ema + (1-d)*buf
        eng = dp.module.__dict__.get('_engine')
        if eng is not None:
            eng.weights_changed()            # weights changed through the flat buffer: re-pack on the next forward

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        tiles = self._tile_table()
        hp, ema, d = self._step_common()
        for gi, group in enumerate(self.param_groups):
            self._fill_group(hp.group[gi], group, gi)
        self._launch(tiles, hp, ema)
        self._step_done(ema, d)
        return loss

    def zero_grad(self, set_to_none=True):
        """One memset of the flat gradient.  `.grad` stays the flat view the training plan writes into, whatever
        set_to_none says."""
        self.dp.flat_grad.zero_()

    def state_dict(self):
        sd = super().state_dict()
        sd['state'] = {k: {kk: (vv.clone() if torch.is_tensor(vv) else vv) for kk, vv in v.items()}
                       for k, v in sd['state'].items()}
        return sd

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)          # checks the group structure, takes the saved hyper-parameters
        loaded, self.state = self.state, defaultdict(dict)
        per_param = [loaded.get(p, {}) for p in self.dp.params]
        if not any(per_param):
            self._reset_state()
            return
        if not all(per_param):
            raise ValueError("optimizer state covers only some parameters; the flat optimiser steps all of them")
        self._load_state(per_param)

    def _copy_flat(self, flat, tensors):
        flat.copy_(torch.cat([t.reshape(-1).to(device=flat.device, dtype=flat.dtype) for t in tensors]))


def build_tile_table(dp, param_groups):
    """The tile table of an optimiser over dp with these groups (see _FlatOptimizer._tile_table); returned on dp's
    device.  Checks that the groups hold each of dp's parameters exactly once."""
    if len(param_groups) > lib.OPT_MAX_GROUPS:
        raise ValueError("at most %d parameter groups" % lib.OPT_MAX_GROUPS)
    owner = {}
    for gi, group in enumerate(param_groups):
        for p in group['params']:
            if id(p) in owner:
                raise ValueError("a parameter is in two groups")
            owner[id(p)] = gi
    if len(owner) != len(dp.params) or any(id(p) not in owner for p in dp.params):
        raise ValueError("the parameter groups must hold exactly the FlatDataParallel's parameters")
    l1_rows = dict(dp._l1[0].tolist()) if dp._l1 is not None else {}
    T = lib.OPT_TILE
    rows, off = [], 0
    for p in dp.params:
        n = p.numel()
        flags = owner[id(p)]
        if off in l1_rows:
            if l1_rows.pop(off) != n:
                raise ValueError("a BatchNorm-L1 range does not cover one whole parameter")
            flags |= lib.OPT_TILE_L1
        s, end = off, off + n
        while s < end:
            e = min(end, (s // T + 1) * T)
            rows.append((s, (e - s) | (flags << 32)))
            s = e
        off = end
    if l1_rows:
        raise ValueError("a BatchNorm-L1 range does not start at a parameter")
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 2).to(dp.flat_param.device)


class FlatSGD(_FlatOptimizer, torch.optim.SGD):
    """torch.optim.SGD (nesterov=True, dampening=0) over dp's flat buffers; `params` is a list of dp's parameters or
    of group dicts, as for torch.optim.SGD."""

    def __init__(self, dp, params, lr, momentum=0.0, dampening=0, weight_decay=0, nesterov=True):
        self._flat_init(dp)
        self._bound = False
        torch.optim.SGD.__init__(self, params, lr=lr, momentum=momentum, dampening=dampening,
                                 weight_decay=weight_decay, nesterov=nesterov)

    def _fill_group(self, G, group, gi):
        if not group['nesterov'] or group['dampening'] != 0 or group['maximize']:
            raise NotImplementedError("FlatSGD implements nesterov=True, dampening=0, maximize=False (train.py:142)")
        G.lr, G.momentum, G.weight_decay = float(group['lr']), float(group['momentum']), float(group['weight_decay'])

    def _launch(self, tiles, hp, ema):
        dp = self.dp
        hp.first_step = 0 if dp.has_momentum else 1
        ops.sgd_grouped(dp.flat_param, dp.flat_grad, dp.flat_mom, tiles, hp, ema=ema)
        dp.has_momentum = True
        if not self._bound:
            self._bind_state()

    def _bind_state(self):
        off = 0
        for p in self.dp.params:
            self.state[p]['momentum_buffer'] = self.dp.flat_mom[off:off + p.numel()].view_as(p)
            off += p.numel()
        self._bound = True

    def _reset_state(self):
        self.dp.has_momentum = False
        self._bound = False

    def _load_state(self, per_param):
        if any(s.get('momentum_buffer') is None for s in per_param):
            raise ValueError("optimizer state without a momentum_buffer")
        self._copy_flat(self.dp.flat_mom, [s['momentum_buffer'] for s in per_param])
        self.dp.has_momentum = True
        self._bind_state()


class FlatAdam(_FlatOptimizer, torch.optim.Adam):
    """torch.optim.Adam (amsgrad=False, L2 weight decay) over dp's flat buffers.  exp_avg / exp_avg_sq are flat buffers
    of their own; each parameter's 'step' is an element of one CPU tensor, so a step advances them all with one op."""

    def __init__(self, dp, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        self._flat_init(dp)
        torch.optim.Adam.__init__(self, params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        self.exp_avg = torch.zeros_like(dp.flat_param)
        self.exp_avg_sq = torch.zeros_like(dp.flat_param)
        self._steps = torch.zeros(len(dp.params), dtype=torch.float32)
        self._index = {id(p): i for i, p in enumerate(dp.params)}
        self._bound = False

    def _fill_group(self, G, group, gi):
        if group['amsgrad'] or group['maximize'] or group.get('decoupled_weight_decay', False):
            raise NotImplementedError("FlatAdam implements amsgrad=False, maximize=False, L2 weight decay")
        if not group['params']:
            return
        t = float(self._steps[self._index[id(group['params'][0])]]) + 1.0
        beta1, beta2 = (float(b) for b in group['betas'])
        lr = float(group['lr'])
        G.weight_decay, G.eps = float(group['weight_decay']), float(group['eps'])
        G.one_minus_beta1, G.beta2, G.one_minus_beta2 = 1.0 - beta1, beta2, 1.0 - beta2
        G.step_size = lr / (1.0 - beta1 ** t)
        G.bc2_sqrt = (1.0 - beta2 ** t) ** 0.5

    def _launch(self, tiles, hp, ema):
        dp = self.dp
        ops.adam_grouped(dp.flat_param, dp.flat_grad, self.exp_avg, self.exp_avg_sq, tiles, hp, ema=ema)
        self._steps += 1
        if not self._bound:
            self._bind_state()

    def _bind_state(self):
        off = 0
        for i, p in enumerate(self.dp.params):
            n = p.numel()
            self.state[p].update(step=self._steps[i], exp_avg=self.exp_avg[off:off + n].view_as(p),
                                 exp_avg_sq=self.exp_avg_sq[off:off + n].view_as(p))
            off += n
        self._bound = True

    def _reset_state(self):
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        self._steps.zero_()
        self._bound = False

    def _load_state(self, per_param):
        steps = torch.tensor([float(s['step']) for s in per_param], dtype=torch.float32)
        for group in self.param_groups:
            idx = [self._index[id(p)] for p in group['params']]
            if idx and not bool((steps[idx] == steps[idx[0]]).all()):
                raise ValueError("the parameters of one group are at different Adam steps")
        self._steps.copy_(steps)
        self._copy_flat(self.exp_avg, [s['exp_avg'] for s in per_param])
        self._copy_flat(self.exp_avg_sq, [s['exp_avg_sq'] for s in per_param])
        self._bind_state()


def make_optimizer(dp, hyp, adam=False, quantized=-1):
    """train.py:120-150 on the flat buffers: FlatAdam(lr0 * 0.005) for --adam and every QAT run (quantized != -1),
    FlatSGD(lr0, momentum, nesterov) otherwise; groups pg0, [pg3], pg1 (weight_decay), pg2."""
    pg0, pg1, pg2, pg3 = train_param_groups(dp, quantized)
    if adam or quantized != -1:
        optimizer = FlatAdam(dp, pg0, lr=hyp['lr0'] * 0.005)
        if quantized == 2:
            optimizer.add_param_group({'params': pg3})
    else:
        optimizer = FlatSGD(dp, pg0, lr=hyp['lr0'], momentum=hyp['momentum'], nesterov=True)
    optimizer.add_param_group({'params': pg1, 'weight_decay': hyp['weight_decay']})
    optimizer.add_param_group({'params': pg2})
    return optimizer
