"""Adaptive quantisation (calcAdaptiveQuantFrame) at 1080p and 2160p, 8 and 10 bit, 4:2:0, aq-mode 2 at qgSize 32 and 8.
Reports, per configuration:
  * the device pass (x265cu_aq_energy): CUDA events around the launch, 3 warm-ups, median of 20; the compulsory bytes
    (1.5 * W * H * bytes per sample: every sample of the three planes read once) and the rate they imply;
  * the host finish (x265cu_aq_finish) on the downloaded energies and totals: host clock, 3 warm-ups, median of 20;
  * the reference calcAdaptiveQuantFrame on one host thread (oracle/_ref/libx265ref_aq{8,10}.so, including the shim's
    Frame set-up; skipped where it is not built);
  * the card name and its power limit."""
import ctypes as C
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import aq_helpers as A  # noqa: E402
import x265_b200  # noqa: E402
from x265_b200.lib import AqOut, AqParams  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    cu = x265_b200.load()
    print("card: %s" % card())
    for (W, H) in [(1920, 1080), (3840, 2160)]:
        for depth in (8, 10):
            pic = A.picture(W, H, depth, "smooth")
            d = [cu.to_device(p) for p in pic]
            B = 1 if depth == 8 else 2
            for qg in (32, 8):
                nb, count, n8 = A.geometry(W, H, qg)
                e, t = cu.alloc(4 * nb), cu.alloc(48)
                dev = []
                for it in range(23):
                    cu.timer_begin()
                    assert cu.L.x265cu_aq_energy(cu.ctx, depth, d[0].ptr, W, d[1].ptr, d[2].ptr, W // 2, W, H, qg, e.ptr, t.ptr) == 0
                    ms = cu.timer_end()
                    if it >= 3:
                        dev.append(ms)
                he, ht = e.download(np.uint32, nb), t.download(np.uint64, 6)
                oe, ot = A.oracle_energy(pic, W, H, depth, qg)
                assert np.array_equal(he, oe) and np.array_equal(ht, ot)
                p = AqParams(aqMode=2, qgSize=qg, weightp=1, aqStrength=1.0)
                qp, iq, iq8 = np.zeros(count), np.zeros(count, np.int32), np.zeros(n8, np.int32)
                ws, wd = np.zeros(3, np.uint64), np.zeros(3, np.uint64)
                out = AqOut(qp.ctypes.data, iq.ctypes.data, iq8.ctypes.data if qg == 8 else None, ws.ctypes.data, wd.ctypes.data,
                            None, None)
                host = []
                for it in range(23):
                    t0 = time.perf_counter()
                    assert cu.L.x265cu_aq_finish(depth, W, H, C.byref(p), he.ctypes.data, ht.ctypes.data, C.byref(out)) == 0
                    if it >= 3:
                        host.append((time.perf_counter() - t0) * 1e3)
                byts = 1.5 * W * H * B
                md = statistics.median(dev)
                line = ("%dx%d %2d-bit qg%-2d  device pass: median %.4f ms (min %.4f, max %.4f), %.1f MB compulsory, %.0f GB/s;"
                        "  host finish: median %.3f ms" % (W, H, depth, qg, md, min(dev), max(dev), byts / 1e6, byts / md / 1e6,
                                                          statistics.median(host)))
                if A.load_ref_aq(depth) is not None:
                    rt = []
                    prm = (2, 1.0, qg, 1, 0, 0)
                    for _ in range(3):
                        t0 = time.perf_counter()
                        A.reference(pic, W, H, depth, prm)
                        rt.append((time.perf_counter() - t0) * 1e3)
                    line += ";  reference, one host thread: median %.1f ms" % statistics.median(rt)
                print(line, flush=True)
                e.free(); t.free()
            for b in d:
                b.free()


if __name__ == "__main__":
    main()
