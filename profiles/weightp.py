"""Weighted-prediction analysis (weightAnalyse) at 2160p 8-bit P, 2160p 10-bit B (two lists) and 1080p 8-bit P, 4:2:0,
on a fade of moving textured content with the lookahead's motion fields, where the search weights luma and so also
costs both chroma planes of every list (a weighted frame's whole work).  Reports, per configuration:
  * the device analysis (x265cu_weightp_analyse: every cost launch, download and the host search): CUDA events around
    the call, 3 warm-ups, median of 20, the kernel launches one call makes (one per costed plane and list: list 1's
    chroma can stop early) and the resulting list-0 luma weights;
  * the reference weightAnalyse on one host thread (oracle/_ref/libx265ref_weightp{8,10}.so; the time includes the
    shim's Frame set-up, Lowres::init and lowresIntraEstimate, so it bounds the function from above; skipped where it is
    not built);
  * the card name and its power limit."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import weightp_helpers as WH  # noqa: E402
import x265_b200  # noqa: E402
from x265_b200.lib import WpFrame  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    cu = x265_b200.load()
    res = dict(card=card(), configs=[])
    for case in (WH._case("noise_fade", 3840, 2160, 8, 1, "P", 1, "la"), WH._case("noise_fade", 3840, 2160, 10, 1, "B", 1, "la"),
                 WH._case("noise_fade", 1920, 1080, 8, 1, "P", 1, "la")):
        c = WH.Case(case)
        import test_gpu_weightp as T
        recs, keep, intra, mvs = T._device_records(cu, c)
        refs = (C.POINTER(WpFrame) * 2)(C.pointer(recs[0]), C.pointer(recs[2]) if c.nl == 2 else C.POINTER(WpFrame)())
        mv = (C.c_void_p * 2)(*mvs)
        out = np.zeros((2, 16, 3, 4), np.int32)
        call = lambda: cu.check(cu.L.x265cu_weightp_analyse(cu.ctx, c.depth, C.byref(c.params), C.byref(recs[1]), intra, refs, mv,
                                                            out.ctypes.data))
        for _ in range(3):
            call()
        n0 = cu.launch_count(); call(); launches = cu.launch_count() - n0
        ms = []
        for _ in range(20):
            cu.timer_begin(); call(); ms.append(cu.timer_end())
        want = WH.oracle_table(c, fill=0)
        assert np.array_equal(c.written(out), c.written(want)), case[0]
        assert launches >= 3, (case[0], launches)                     # luma weighted: the chroma planes were costed
        ref_ms = None
        if WH.load_ref_wp(c.depth) is not None:
            t = []
            for _ in range(3):
                t0 = time.perf_counter(); WH.reference_table(c); t.append((time.perf_counter() - t0) * 1e3)
            ref_ms = statistics.median(t)
        r = dict(case=case[0], device_ms=statistics.median(ms), launches=launches,
                 reference_host_ms_with_frame_setup=ref_ms, luma_L0=c.written(out)[0])
        print(json.dumps(r))
        res["configs"].append(r)
    print("card:", res["card"])


if __name__ == "__main__":
    main()
