"""The adaptive-BatchNorm recalibration of tests/golden/pruned_adabn_case.npz (oracle/gen_golden_adabn.py): the pruned
fixture models in train mode, three gradient-free forwards, then eval.  `rows` is the generator's subsample of p / io."""
import torch

from helpers import golden, orc
from pruned_models import compact_defs

_G = None
ROWS = 16


def adabn_fixture():
    global _G
    if _G is None:
        _G = golden("pruned_adabn_case")
    return _G


def batches(name):
    g = adabn_fixture()
    size = dict(fixture_cases())[name]
    return [orc.synth_images(int(g["batch"]), size, size, seed=int(s)) for s in g["seeds"]]


def fixture_cases():
    import json
    return [tuple(c) for c in json.loads(str(adabn_fixture()["cases"]))]


def eval_images(name):
    size = dict(fixture_cases())[name]
    return orc.synth_images(2, size, size, seed=5)


def rows(t):
    """[B, ..., no] -> [B, <= ROWS, no]: every step-th output row of each image"""
    t = t.reshape(t.shape[0], -1, t.shape[-1])
    return t[:, ::-(-t.shape[1] // ROWS)]


def oracle_recalibrate(name, state, emulate_fp16=False):
    """p (list per batch of lists per head) of the three recalibration forwards; `state` (cpu state_dict) gets the
    updated running statistics"""
    defs = compact_defs(name)[1:]
    ps = []
    for x in batches(name):
        with torch.no_grad():
            p, new_stats = orc.darknet_forward(defs, state, x, name, training=True, emulate_fp16=emulate_fp16)
        state.update(new_stats)
        ps.append(p)
    return ps


def stat_keys(name):
    return [k[len(name) + 7:] for k in adabn_fixture().files if k.startswith(name + ":stat::")]

