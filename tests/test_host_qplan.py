"""CPU: the decisions the INT8 graph (qengine.QPlan) and the fp16 eval plan (engine.Plan) take when they are built: the
kinds of the steps, which convs carry a folded shortcut, and the pixel-pair form of every conv (layout.pair_form),
pinned per cfg and input size; and pair_form itself on the edges of its shape rule."""
import pytest
import torch

from helpers import cfg_path

CPU = torch.device("cpu")
SIZES = [(416, 416), (96, 64)]

# one letter per step: c conv, s shortcut, r concat, u upsample, m maxpool
YOLOV3_KINDS = "ccccccccccccccccccccccccccccccccccccccccccccccccccccccccccccurccccccccurccccccc"
YOLOV3_PLAIN_KINDS = ("ccccscccsccscccsccsccsccsccsccsccsccscccsccsccsccsccsccsccsccscccsccsccsccsccccccccurccccccccurcc"
                      "ccccc")
# every shortcut of yolov3 is folded into the conv before it
YOLOV3_FUSED = [3, 7, 10, 14, 17, 20, 23, 26, 29, 32, 35, 39, 42, 45, 48, 51, 54, 57, 60, 64, 67, 70, 73]
YOLOV3_FORMS = {1: 's2', 3: 's1'}

INT8_CASES = {
    # (cfg, quantized, shortcut_way): (kinds, convs with a folded shortcut, {conv: form} of the paired convs)
    ("yolov3", 3, 1): (YOLOV3_KINDS, YOLOV3_FUSED, YOLOV3_FORMS),
    ("yolov3", 1, 1): (YOLOV3_KINDS, YOLOV3_FUSED, YOLOV3_FORMS),
    ("yolov3", 1, 2): (YOLOV3_KINDS, YOLOV3_FUSED, YOLOV3_FORMS),
    ("yolov3-tiny", 1, 1): ("cmcmcmcmcmcmcccccurcc", [], {4: 's1'}),
    ("yolov3-spp", 1, 1): ("cccccccccccccccccccccccccccccccccccccccccccccccccccccccmmmrccccccurccccccccurccccccc",
                           YOLOV3_FUSED, YOLOV3_FORMS),
}
FP16_FORMS = {"yolov3": YOLOV3_FORMS, "yolov4": {1: 's2', 6: 's1'}, "yolov3-tiny": {4: 's1'}}
_LETTER = {'conv': 'c', 'shortcut': 's', 'concat': 'r', 'upsample': 'u', 'maxpool': 'm'}


def _int8_model(name, quantized, way):
    import models
    import test_gpu_qat_int8 as qi      # the yolov3-spp cfg
    kw = dict(steps=qi.STEPS) if quantized == 1 else {}
    return models.Darknet(qi._cfg(name), quantized=quantized, a_bit=8, w_bit=8, shortcut_way=way, **kw).eval()


def _decisions(plan):
    convs = [st for st in plan.steps if st.kind == 'conv']
    return ("".join(_LETTER[st.kind] for st in plan.steps), [st.i for st in convs if st.shortcut],
            {st.i: st.form for st in convs if st.form is not None})


@pytest.mark.parametrize("case", list(INT8_CASES), ids=lambda c: "%s-q%d-way%d" % c)
def test_int8_plan_decisions(case):
    from b200yolo.qengine import QPlan
    model = _int8_model(*case)
    for h, w in SIZES:
        assert _decisions(QPlan(model, (2, 3, h, w), CPU)) == INT8_CASES[case], (h, w)


def test_int8_plain_plan():
    """pair_forms=False, fuse_shortcuts=False: dense weights and a launch of its own for every shortcut"""
    from b200yolo.qengine import QPlan
    model = _int8_model("yolov3", 3, 1)
    for h, w in SIZES:
        plan = QPlan(model, (2, 3, h, w), CPU, pair_forms=False, fuse_shortcuts=False)
        assert _decisions(plan) == (YOLOV3_PLAIN_KINDS, [], {}), (h, w)


@pytest.mark.parametrize("name", list(FP16_FORMS))
def test_fp16_plan_forms(name):
    import models
    from b200yolo.engine import Plan
    model = models.Darknet(cfg_path(name)).eval()
    for h, w in SIZES:
        plan = Plan(model, (2, 3, h, w), CPU)
        assert {st.i: st.form for st in plan.steps if st.kind == 'conv' and st.form} == FP16_FORMS[name], (h, w)


@pytest.mark.parametrize("shape,form", [
    ((3, 1, 1, 32, 64, 64), 's1'),
    ((3, 1, 1, 32, 128, 64), 's1'),
    ((3, 1, 1, 32, 120, 64), 's1'),
    ((3, 1, 1, 32, 136, 64), None),
    ((3, 1, 1, 32, 12, 64), None),
    ((3, 1, 1, 32, 64, 63), None),          # odd width: no whole pixel pairs
    ((3, 2, 1, 32, 64, 63), None),
    ((3, 1, 0, 32, 64, 64), None),
    ((3, 2, 0, 32, 64, 64), None),
    ((3, 2, 1, 32, 64, 64), 's2'),
    ((3, 2, 1, 32, 256, 64), 's2'),         # stride 2: any output width
    ((3, 1, 1, 64, 64, 64), None),
    ((1, 1, 0, 32, 64, 64), None),
    ((3, 3, 1, 32, 64, 64), None),
])
def test_pair_form(shape, form):
    from b200yolo.layout import pair_form
    assert pair_form(*shape) == form
