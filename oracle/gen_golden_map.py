"""Generate tests/golden/map_case.npz by RUNNING THE REFERENCE (CPU): yolov3-tiny eval forward on a seeded batch,
the reference's non_max_suppression / clip_coords / test.py matching loop / ap_per_class.  The reference's own
detections (conf > 0.3) are the held labels, so its mAP is the self-consistency value of the pipeline; the H100 engine
must reproduce that mAP within 1e-4 from ITS predictions (tests/test_gpu_model.py), and oracle/metrics_oracle.py is pinned
against every intermediate stored here (tests/test_oracle_golden.py).

    python oracle/gen_golden_map.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("B2Y_REFERENCE_ROOT", "/root/reference")
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "mpl_stub"))
os.chdir(REF)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import models as ref_models  # noqa: E402  (the reference)
from utils import utils as ru  # noqa: E402

sys.path.insert(0, HERE)
import darknet_oracle as orc  # noqa: E402

NAME, CFG, B, S, SEED = "yolov3-tiny", "cfg/yolov3tiny/yolov3-tiny.cfg", 2, 416, 7
CONF, IOU = 0.3, 0.6


def main():
    model = ref_models.Darknet(CFG, img_size=(S, S))
    model.load_state_dict(orc.synth_state_dict(model.state_dict(), 0))
    model.eval()
    x = orc.synth_images(B, S, S, seed=SEED)
    with torch.no_grad():
        inf_out = model(x)[0]
    dets = ru.non_max_suppression(inf_out.clone(), conf_thres=CONF, iou_thres=IOU)
    iouv = torch.linspace(0.5, 0.95, 10)
    niou = iouv.numel()
    for d in dets:
        ru.clip_coords(d, (S, S))
    labels = [torch.cat((d[:, 5:6], d[:, :4]), 1).clone() for d in dets]          # (cls, xyxy)
    stats = []
    for pred, lab in zip(dets, labels):                                            # test.py:123-175
        tcls = lab[:, 0].tolist()
        correct = torch.zeros(pred.shape[0], niou, dtype=torch.bool)
        detected = []
        tcls_tensor = lab[:, 0]
        tbox = lab[:, 1:5]
        for cls in torch.unique(tcls_tensor):
            ti = (cls == tcls_tensor).nonzero(as_tuple=False).view(-1)
            pi = (cls == pred[:, 5]).nonzero(as_tuple=False).view(-1)
            if pi.shape[0]:
                ious, i = ru.box_iou(pred[pi, :4], tbox[ti]).max(1)
                for j in (ious > iouv[0]).nonzero(as_tuple=False):
                    d = ti[i[j]]
                    if d not in detected:
                        detected.append(d)
                        correct[pi[j]] = ious[j] > iouv
                        if len(detected) == len(lab):
                            break
        stats.append((correct, pred[:, 4], pred[:, 5], tcls))
    cols = [np.concatenate([np.asarray(t) for t in c], 0) for c in zip(*stats)]
    p, r, ap, f1, ap_class = ru.ap_per_class(*cols)
    out = {"inf_out": inf_out.numpy(), "conf_thres": np.float32(CONF), "iou_thres": np.float32(IOU),
           "size": np.int32(S), "seed": np.int32(SEED), "map50": np.float64(ap[:, 0].mean()),
           "map": np.float64(ap.mean(1).mean()), "ap": ap, "ap_class": ap_class, "p": p, "r": r}
    for i, (d, lab) in enumerate(zip(dets, labels)):
        out["det%d" % i] = d.numpy()
        out["labels%d" % i] = lab.numpy()
        out["correct%d" % i] = stats[i][0].numpy()
    path = os.path.join(ROOT, "tests", "golden", "map_case.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; detections", [d.shape[0] for d in dets], "mAP50 %.6f mAP %.6f"
          % (out["map50"], out["map"]))


if __name__ == "__main__":
    main()
