"""Generate tests/golden/ref_cfg_layers.json from the reference's own .cfg files: the layer fields that
tests/test_host.py compares with the generated cfgs (b200yolo/cfggen.py), as parsed by the reference's own cfg parser
(utils/parse_config.py of the reference), so that a bug in this package's parser cannot cancel out.

    python oracle/gen_golden_cfg.py /path/to/reference
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CFGS = {"yolov3": "cfg/yolov3/yolov3.cfg", "yolov3-tiny": "cfg/yolov3tiny/yolov3-tiny.cfg",
        "yolov4": "cfg/yolov4/yolov4.cfg", "yolov3-mobilenet": "cfg/yolov3-mobilenet/yolov3-mobilenet-coco.cfg"}
KEYS = ('type', 'batch_normalize', 'filters', 'size', 'stride', 'pad', 'activation', 'layers', 'from', 'mask',
        'classes', 'num', 'anchors')


def _plain(v):
    if hasattr(v, "tolist"):
        return v.tolist()
    return v


def main(ref):
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_parse_config", os.path.join(ref, "utils", "parse_config.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    parse_model_cfg = mod.parse_model_cfg
    out = {}
    for name, rel in CFGS.items():
        defs = parse_model_cfg(os.path.join(ref, rel))[1:]
        out[name] = [{k: _plain(d[k]) for k in KEYS if k in d} for d in defs]
    path = os.path.join(ROOT, "tests", "golden", "ref_cfg_layers.json")
    with open(path, "w") as f:
        json.dump(out, f, sort_keys=True, separators=(",", ":"))
    print(path)


if __name__ == "__main__":
    main(sys.argv[1])
