"""The reference's optimiser and burn-in (train.py:120-144, :356-365) restated over plain torch.optim, for the tests of
b200yolo.optim."""
import math

import numpy as np
import torch

HYP = {'lr0': 0.01, 'momentum': 0.937, 'weight_decay': 0.0005}


def group_of(name, quantized):
    """train.py:126-133: which of pg0 / pg1 / pg2 / pg3 a parameter name goes to (first matching test wins)."""
    if '.bias' in name:
        return 'pg2'
    if 'Conv2d.weight' in name:
        return 'pg1'
    if 'scale' in name and quantized == 2:
        return 'pg3'
    return 'pg0'


def torch_optimizer(model, hyp=HYP, adam=False, quantized=-1):
    """torch.optim.SGD / Adam over `model`'s parameters, built the way train.py:120-144 builds it."""
    pg = {'pg0': [], 'pg1': [], 'pg2': [], 'pg3': []}
    for k, v in dict(model.named_parameters()).items():
        pg[group_of(k, quantized)].append(v)
    if adam or quantized != -1:
        opt = torch.optim.Adam(pg['pg0'], lr=hyp['lr0'] * 0.005)
        if quantized == 2:
            opt.add_param_group({'params': pg['pg3']})
    else:
        opt = torch.optim.SGD(pg['pg0'], lr=hyp['lr0'], momentum=hyp['momentum'], nesterov=True)
    opt.add_param_group({'params': pg['pg1'], 'weight_decay': hyp['weight_decay']})
    opt.add_param_group({'params': pg['pg2']})
    return opt


def cosine_lf(epochs):
    """train.py:201, the LambdaLR factor."""
    return lambda x: (((1 + math.cos(x * math.pi / epochs)) / 2) ** 1.0) * 0.95 + 0.05


def burn_in(optimizer, ni, n_burn, epoch, lf, hyp=HYP):
    """train.py:356-365 for iteration ni (applied while ni <= n_burn)."""
    xi = [0, n_burn]
    for j, x in enumerate(optimizer.param_groups):
        x['lr'] = np.interp(ni, xi, [0.1 if j == 2 else 0.0, x['initial_lr'] * lf(epoch)])
        x['weight_decay'] = np.interp(ni, xi, [0.0, hyp['weight_decay'] if j == 1 else 0.0])
        if 'momentum' in x:
            x['momentum'] = np.interp(ni, xi, [0.9, hyp['momentum']])
