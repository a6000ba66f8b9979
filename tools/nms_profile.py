"""Run the bench's NMS + TP-matching block a few times (for an ncu launch list of csrc/nms.cu):

    ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none --csv \\
        --log-file launches_nms.csv python tools/nms_profile.py
"""
import os
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "yolov3v4-modelcompression-multidatasettraining-multibackbone_b200"))
import torch  # noqa: E402

import bench  # noqa: E402

if __name__ == "__main__":
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = bench.run_nms(SimpleNamespace(steps=3), dev, bench.Dist(1, dev))
    print(out)
