"""cuTree's propagation chain on the device (x265cu_cutree) over a 2160p preset-slow window: 40 frames of lookahead (41
frames), bframes 4 with b-pyramid (param.cpp: preset slow).  Inputs are synthetic estimates of the real shapes.  Reports:
  * the device chain time: CUDA events around x265cu_cutree, warm-up, median of 20;
  * the reference Lookahead::cuTree on one host thread over the same inputs (oracle/_ref/libx265ref_cutree8.so; skipped
    where it is not built);
  * the bytes a host cuTree needs downloaded (every estimate's lowresCosts and motion fields, intraCost, invQscale)
    against the bytes Lookahead.cu_tree downloads (the finished frames' propagateCost);
  * the card name and its power limit."""
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import cutree_helpers as T  # noqa: E402
import x265_b200  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    from test_gpu_cutree import DeviceWindow
    cu = x265_b200.load()
    w8, h8 = 240, 135
    types = T.slice_types(41, 4)
    prm = T.params(bBPyramid=1)
    win = T.synth_window(cu, "profile", w8, h8, types, prm)
    d = DeviceWindow(cu, win)
    import ctypes as C
    fin = np.zeros(2 * (win.n + 2), np.int32)
    times = []
    for it in range(25):
        d.reset()
        cu.sync()
        cu.timer_begin()
        assert cu.L.x265cu_cutree(cu.ctx, d.recs, win.n - 1, C.byref(d.prm), w8, h8, fin.ctypes.data, win.n + 2) >= 0
        ms = cu.timer_end()
        if it >= 5:
            times.append(ms)
    print("card: %s" % card())
    print("device chain, 2160p, 41-frame window, bframes 4 + b-pyramid: median %.3f ms over 20 (min %.3f, max %.3f)"
          % (statistics.median(times), min(times), max(times)))
    host_bytes = sum(a.nbytes for a in win.costs.values()) + sum(a.nbytes for a in win.mvs.values()) + \
        sum(win.intra[f].nbytes + win.invq[f].nbytes for f in range(win.n))
    nfin = len([1 for _, dd in d.run()[1] if dd >= 0])
    print("host cuTree download: %.2f MB; device chain download: %.3f MB (%d finished frames' propagateCost)"
          % (host_bytes / 1e6, nfin * 2 * w8 * h8 / 1e6, nfin))
    if T.load_ref_cutree(8) is not None:
        rt = []
        for _ in range(5):
            t0 = time.perf_counter()
            win.reference()
            rt.append((time.perf_counter() - t0) * 1e3)
        print("reference Lookahead::cuTree, one host thread (incl. the shim's set-up): median %.2f ms" % statistics.median(rt))
    else:
        print("reference Lookahead::cuTree: not measured (oracle/_ref not built)")
    d.close()


if __name__ == "__main__":
    main()
