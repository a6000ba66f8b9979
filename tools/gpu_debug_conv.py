"""Debug driver (not a pytest file): run conv parity cases one process per case so that a trapped kernel
(bounded mbarrier wait -> __trap) cannot poison the following cases.  Usage on a GPU machine:
    python tests/gpu_debug_conv.py            # all cases, one subprocess each
    python tests/gpu_debug_conv.py 3          # a single case in-process
"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conftest  # noqa: F401  (sets sys.path)


def main():
    from test_gpu_kernels import CONV_CASES, conv_case
    if len(sys.argv) > 1:
        i = int(sys.argv[1])
        err, rms = conv_case(*CONV_CASES[i])
        print("CASE %d %s err=%.4g rms=%.4g rel=%.3g" % (i, CONV_CASES[i], err, rms, err / max(rms, 1e-9)), flush=True)
        return
    for i in range(len(CONV_CASES)):
        r = subprocess.run([sys.executable, __file__, str(i)], capture_output=True, text=True, timeout=300)
        tail = (r.stdout.strip().splitlines() or [""])[-1]
        if r.returncode != 0:
            tail = "FAILED rc=%d: %s" % (r.returncode, (r.stderr.strip().splitlines() or [""])[-1])
        print("[%d] %s" % (i, tail), flush=True)


if __name__ == "__main__":
    main()
